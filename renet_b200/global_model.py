"""The global model of RE-Net (reference global_model.py + Aggregator.RGCNAggregator_global, Aggregator.py:9-107) on the
sm_90a kernels -- SURVEY.md section 8(f) row 4.  It produces the ``global_emb[t]`` vectors the hot path consumes
(utils.py:224-225) and is pre-trained by the reference's pretrain.py.

Same class surface as the reference (constructor signatures, attribute / parameter names, so ``state_dict`` keys carry
over: ``ent_embeds``, ``encoder_global.*``, ``aggregator.rgcn{1,2}.*``, ``linear_s.*``, ``linear_o.*``):

    RGCNAggregator_global(h_dim, dropout, num_nodes, num_rels, num_bases, model, seq_len=10, maxpool=1)
        .forward(t_list, ent_embeds, graph_dict, reverse) -> PackedSequence   (Aggregator.py:27-73)
        .predict(t, ent_embeds, graph_dict, reverse) -> [len, h]             (Aggregator.py:75-107)
    RENet_global(in_dim, h_dim, num_rels, dropout=0, model=0, seq_len=10, num_k=10, maxpool=1)
        .forward(t_list, true_prob_s, true_prob_o, graph_dict, subject=True) -> loss   (global_model.py:35-55)
        .get_global_emb(t_list, graph_dict), .predict(t, graph_dict, subject=True)     (global_model.py:57-92)

What runs where: the whole per-timestamp graphs of the needed timestamps are batched (numpy concatenation of the
destination-sorted per-timestamp edge lists: the batched graph is born in CSR form), both RGCN layers are the fused
kernels of rgcn.py, ``dgl.max_nodes`` / ``mean_nodes`` is renet_segment_pool_fwd/_bwd, and ``encoder_global``
(nn.GRU(h, h): parameter holder) runs through renet_gru_dense_fwd/_bwd (tensor-core input projection + the recurrence
kernel of the hot path).  The two small linear heads and the fp64 soft cross-entropy (utils.py:287-290) stay PyTorch.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.utils.rnn import PackedSequence

from . import _lib
from .graph import BatchedHistoryGraph, as_history_graph
from .rgcn import RGCNBlockLayer as RGCNLayer


def soft_cross_entropy(pred, soft_targets):
    """Reference utils.py:287-290 (fp64 log-softmax, mean over rows of the soft-target cross-entropy)."""
    logp = F.log_softmax(pred.double(), dim=1)
    return torch.mean(torch.sum(-soft_targets.double() * logp, 1))


def whole_graph_arrays(graphs):
    """Host half of dgl.batch over WHOLE per-timestamp graphs (Aggregator.py:53,96): every per-timestamp edge list is
    destination-sorted, so concatenation with node offsets IS the CSR of the batched graph.  Returns numpy arrays
    (node_ent, norm, row_ptr, col_src, col_type_s, col_type_o, sizes, node offsets [G+1])."""
    graphs = [as_history_graph(g) for g in graphs]
    sizes = np.asarray([g.number_of_nodes() for g in graphs], dtype=np.int64)
    off = np.concatenate(([0], np.cumsum(sizes)))
    node_ent = np.concatenate([g.node_id for g in graphs])
    norm = np.concatenate([g.norm for g in graphs])
    src = np.concatenate([g.src.astype(np.int64) + o for g, o in zip(graphs, off[:-1])])
    dst = np.concatenate([g.dst.astype(np.int64) + o for g, o in zip(graphs, off[:-1])])
    row_ptr = np.concatenate(([0], np.cumsum(np.bincount(dst, minlength=int(off[-1])))))
    return (node_ent, norm, row_ptr, src, np.concatenate([g.type_s for g in graphs]),
            np.concatenate([g.type_o for g in graphs]), sizes, off)


def batch_whole_graphs(graphs, device):
    """dgl.batch + move_dgl_to_cuda of whole graphs: BatchedHistoryGraph + node offsets [G+1] on the device."""
    node_ent, norm, row_ptr, src, ts, to, sizes, off = whole_graph_arrays(graphs)
    bg = BatchedHistoryGraph(node_ent, norm, row_ptr, src, ts, to, sizes, device)
    seg = torch.from_numpy(off.astype(np.int32)).to(device)
    return bg, seg


class _SegmentPoolFn(torch.autograd.Function):
    """dgl.max_nodes / mean_nodes (Aggregator.py:58-61)."""

    @staticmethod
    def forward(ctx, H, seg_ptr, mode):
        L, P = _lib.lib(), _lib.ptr
        _lib.require_cuda(H, seg_ptr)
        H = H.contiguous()
        G, d = seg_ptr.numel() - 1, H.shape[1]
        out = torch.empty(G, d, device=H.device)
        arg = torch.empty(G, d, dtype=torch.int32, device=H.device) if mode == 1 else None
        _lib.check(L.renet_segment_pool_fwd(P(H), P(seg_ptr), G, d, mode, P(out), P(arg), _lib.stream()), 'renet_segment_pool_fwd')
        ctx.save_for_backward(seg_ptr, arg if arg is not None else seg_ptr)
        ctx.mode, ctx.N = mode, H.shape[0]
        return out

    @staticmethod
    def backward(ctx, dout):
        L, P = _lib.lib(), _lib.ptr
        seg_ptr, arg = ctx.saved_tensors
        dout = dout.contiguous()
        G, d = dout.shape
        dH = torch.empty(ctx.N, d, device=dout.device)
        _lib.check(L.renet_segment_pool_bwd(P(dout), P(seg_ptr), P(arg) if ctx.mode == 1 else None, G, ctx.N, d, ctx.mode, P(dH),
                                            _lib.stream()), 'renet_segment_pool_bwd')
        return dH, None, None


class _DenseGruFn(torch.autograd.Function):
    """Final hidden state of a 1-layer GRU over sequence-major rows X [S,k] (lengths sorted descending, h0 = 0)."""

    @staticmethod
    def forward(ctx, X, w_ih, w_hh, b_ih, b_hh, seq_len_dev, seq_start_dev, batch_sizes):
        L, P = _lib.lib(), _lib.ptr
        tensors = [t.contiguous() for t in (X, w_ih, w_hh, b_ih, b_hh)]
        _lib.require_cuda(*tensors)
        X, w_ih, w_hh, b_ih, b_hh = tensors
        S, k = X.shape
        h = w_hh.shape[1]
        Q = seq_len_dev.numel()
        dev = X.device
        hn = torch.zeros(2, Q, h, device=dev)
        nbytes = int(L.renet_gru_dropout_workspace_bytes(S, Q, 1, h))
        ws = torch.empty(nbytes // 4 + 32, dtype=torch.float32, device=dev)
        bs = np.ascontiguousarray(batch_sizes, dtype=np.int32)
        rc = L.renet_gru_dense_fwd(P(X), k, None, 0, P(seq_len_dev), P(seq_start_dev), bs.ctypes.data_as(_lib.ctypes.c_void_p),
                                   len(bs), P(w_ih), P(w_hh), P(b_ih), P(b_hh), None, None, None, None, P(hn[0]), P(hn[1]), S, Q,
                                   h, P(ws), nbytes, _lib.stream())
        _lib.check(rc, 'renet_gru_dense_fwd')
        ctx.save_for_backward(X, w_ih, w_hh, seq_len_dev, seq_start_dev, ws)
        ctx.bs = bs
        return hn[0]

    @staticmethod
    def backward(ctx, dhn):
        L, P = _lib.lib(), _lib.ptr
        X, w_ih, w_hh, seq_len_dev, seq_start_dev, ws = ctx.saved_tensors
        S, k = X.shape
        h = w_hh.shape[1]
        Q = seq_len_dev.numel()
        dev = X.device
        dhn = dhn.contiguous()
        zero = torch.zeros_like(dhn)
        dX = torch.empty_like(X)
        dw_ih, dw_hh = torch.zeros_like(w_ih), torch.zeros_like(w_hh)
        db_ih, db_hh = torch.zeros(3 * h, device=dev), torch.zeros(3 * h, device=dev)
        nbytes = int(L.renet_gru_bwd_dropout_workspace_bytes(S, Q, 1, h))
        bws = torch.empty(nbytes // 4 + 32, dtype=torch.float32, device=dev)
        bs = ctx.bs
        rc = L.renet_gru_dense_bwd(P(X), k, None, 0, P(seq_len_dev), P(seq_start_dev), bs.ctypes.data_as(_lib.ctypes.c_void_p),
                                   len(bs), P(w_ih), P(w_hh), None, None, P(dhn), P(zero), P(dX), None, P(dw_ih), P(dw_hh),
                                   P(db_ih), P(db_hh), None, None, None, None, S, Q, h, P(ws), P(bws), nbytes, _lib.stream())
        _lib.check(rc, 'renet_gru_dense_bwd')
        return dX, dw_ih, dw_hh, db_ih, db_hh, None, None, None


def gru_final_hidden(gru, X, seq_len):
    """``gru``: nn.GRU(k, h) parameter holder; X [S,k] sequence-major rows; seq_len: host int array sorted descending."""
    if gru.num_layers != 1 or gru.bidirectional or not gru.bias:
        raise RuntimeError('renet_b200 dense GRU supports 1 layer, unidirectional, with bias (global_model.py:25)')
    seq_len = np.asarray(seq_len, dtype=np.int64)
    dev = X.device
    start = np.concatenate(([0], np.cumsum(seq_len)[:-1])).astype(np.int32)
    max_len = int(seq_len[0]) if len(seq_len) else 0
    bs = np.asarray([int(np.count_nonzero(seq_len > t)) for t in range(max_len)], dtype=np.int32)
    both = torch.from_numpy(np.concatenate((seq_len.astype(np.int32), start))).to(dev)
    return _DenseGruFn.apply(X, gru.weight_ih_l0, gru.weight_hh_l0, gru.bias_ih_l0, gru.bias_hh_l0, both[:len(seq_len)],
                             both[len(seq_len):], bs)


class RGCNAggregator_global(nn.Module):
    def __init__(self, h_dim, dropout, num_nodes, num_rels, num_bases, model, seq_len=10, maxpool=1):
        super(RGCNAggregator_global, self).__init__()
        self.h_dim = h_dim
        self.dropout = nn.Dropout(dropout)
        self.seq_len = seq_len
        self.num_rels = num_rels
        self.num_nodes = num_nodes
        self.model = model
        self.maxpool = maxpool
        self.rgcn1 = RGCNLayer(self.h_dim, self.h_dim, 2 * self.num_rels, num_bases,
                               activation=F.relu, self_loop=True, dropout=dropout)
        self.rgcn2 = RGCNLayer(self.h_dim, self.h_dim, 2 * self.num_rels, num_bases,
                               activation=None, self_loop=True, dropout=dropout)

    def _global_info(self, times_needed, ent_embeds, graph_dict, reverse):
        """Aggregator.py:53-62 / 96-105: batch the whole graphs, two RGCN layers, pool per graph -> [G, h]."""
        dev = ent_embeds.device
        bg, seg = batch_whole_graphs([graph_dict[int(t)] for t in times_needed], dev)
        H1 = self.rgcn1.apply_layer(bg, ent_embeds, bg.node_ent, reverse)
        H2 = self.rgcn2.apply_layer(bg, H1, None, reverse)
        return _SegmentPoolFn.apply(H2, seg, 1 if self.maxpool == 1 else 0)

    def _windows(self, t_list, graph_dict):
        """Aggregator.py:28-45: per non-zero t the (<= seq_len) timestamps before it, and their count."""
        times = list(graph_dict.keys())
        time_unit = times[1] - times[0]
        t_host = [int(t) for t in (t_list.tolist() if torch.is_tensor(t_list) else t_list)]
        num_non_zero = sum(1 for t in t_host if t != 0)
        time_list, len_non_zero = [], []
        for tim in t_host[:num_non_zero]:
            length = int(tim // time_unit)
            if self.seq_len <= length:
                time_list.append(times[length - self.seq_len:length])
                len_non_zero.append(self.seq_len)
            else:
                time_list.append(times[:length])
                len_non_zero.append(length)
        return time_list, len_non_zero

    def rows(self, t_list, ent_embeds, graph_dict, reverse):
        """Sequence-major GRU input rows [S,h] (after dropout) and the sequence lengths (Aggregator.py:27-69)."""
        time_list, len_non_zero = self._windows(t_list, graph_dict)
        unique_t = sorted({int(t) for w in time_list for t in w})            # torch.unique sorts (Aggregator.py:47)
        time_to_idx = {t: i for i, t in enumerate(unique_t)}
        info = self._global_info(unique_t, ent_embeds, graph_dict, reverse)
        idx = torch.tensor([time_to_idx[int(t)] for w in time_list for t in w], dtype=torch.long, device=ent_embeds.device)
        return self.dropout(info[idx]), len_non_zero

    def forward(self, t_list, ent_embeds, graph_dict, reverse):
        """Reference Aggregator.py:27-73: returns the PackedSequence of per-timestamp global vectors (time-major)."""
        X, lens = self.rows(t_list, ent_embeds, graph_dict, reverse)
        lens = np.asarray(lens, dtype=np.int64)
        start = np.concatenate(([0], np.cumsum(lens)[:-1]))
        max_len = int(lens.max()) if len(lens) else 0
        bs = np.asarray([int(np.count_nonzero(lens > t)) for t in range(max_len)], dtype=np.int64)
        perm = np.concatenate([start[:bs[t]] + t for t in range(max_len)]) if max_len else np.zeros(0, np.int64)
        return PackedSequence(X[torch.from_numpy(perm).to(X.device)], torch.from_numpy(bs))

    def predict(self, t, ent_embeds, graph_dict, reverse):
        """Reference Aggregator.py:75-107: the pooled vectors of the (<= seq_len) graphs before time t."""
        times = list(graph_dict.keys())
        idx = 0
        for tt in times:
            if tt >= t:
                break
            idx += 1
        window = times[idx - self.seq_len:idx] if self.seq_len <= idx else times[:idx]
        return self._global_info(window, ent_embeds, graph_dict, reverse)


class RENet_global(nn.Module):
    def __init__(self, in_dim, h_dim, num_rels, dropout=0, model=0, seq_len=10, num_k=10, maxpool=1, num_bases=100):
        super(RENet_global, self).__init__()
        self.in_dim = in_dim
        self.h_dim = h_dim
        self.num_rels = num_rels
        self.model = model
        self.seq_len = seq_len
        self.num_k = num_k
        self.ent_embeds = nn.Parameter(torch.Tensor(in_dim, h_dim))
        nn.init.xavier_uniform_(self.ent_embeds, gain=nn.init.calculate_gain('relu'))
        self.dropout = nn.Dropout(dropout)
        self.encoder_global = nn.GRU(h_dim, h_dim, batch_first=True)          # parameters only; math in renet_gru_dense_*
        # the reference hard-codes num_bases = 100 (global_model.py:27); exposed only for small test shapes
        self.aggregator = RGCNAggregator_global(h_dim, dropout, in_dim, num_rels, num_bases, model, seq_len, maxpool)
        self.linear_s = nn.Linear(h_dim, in_dim)
        self.linear_o = nn.Linear(h_dim, in_dim)
        self.global_emb = None

    def forward(self, t_list, true_prob_s, true_prob_o, graph_dict, subject=True):
        """Reference global_model.py:35-55."""
        if subject:
            reverse, linear, true_prob = False, self.linear_s, true_prob_o
        else:
            reverse, linear, true_prob = True, self.linear_o, true_prob_s
        t_host = np.asarray(t_list.tolist() if torch.is_tensor(t_list) else t_list, dtype=np.int64)
        idx = np.argsort(-t_host, kind='stable')                             # t_list.sort(0, descending=True)
        sorted_t = t_host[idx]
        X, lens = self.aggregator.rows(sorted_t, self.ent_embeds, graph_dict, reverse)
        s_q = gru_final_hidden(self.encoder_global, X, lens)
        pad = torch.zeros(len(t_host) - s_q.shape[0], self.h_dim, device=s_q.device)
        s_q = torch.cat((s_q, pad), dim=0)
        pred = linear(s_q)
        return soft_cross_entropy(pred, true_prob[torch.from_numpy(idx).to(true_prob.device)])

    def predict(self, t, graph_dict, subject=True):
        """Reference global_model.py:77-89: (s_q [1,1,h], logits [1,1,in_dim], probabilities [in_dim])."""
        linear, reverse = (self.linear_s, False) if subject else (self.linear_o, True)
        rnn_inp = self.aggregator.predict(t, self.ent_embeds, graph_dict, reverse=reverse)
        s_q = gru_final_hidden(self.encoder_global, rnn_inp, [rnn_inp.shape[0]]).view(1, 1, self.h_dim)
        sub = linear(s_q)
        return s_q, sub, torch.softmax(sub.view(-1), dim=0)

    def get_global_emb(self, t_list, graph_dict):
        """Reference global_model.py:57-73: global_emb[t] for every training timestamp."""
        global_emb = dict()
        times = list(graph_dict.keys())
        time_unit = times[1] - times[0]
        prev_t = 0
        for t in t_list:
            t = int(t)
            if t == 0:
                continue
            emb, _, _ = self.predict(t, graph_dict)
            global_emb[prev_t] = emb.detach()
            prev_t = t
        last, _, _ = self.predict(int(t_list[-1]) + int(time_unit), graph_dict)
        global_emb[int(t_list[-1])] = last.detach()
        return global_emb

    def update_global_emb(self, t, graph_dict):
        pass
