"""RGCNAggregator with the reference's surface (reference Aggregator.py:109-237) on the sm_90a kernels.

Kept verbatim from the reference: constructor signature and attributes, sub-modules ``rgcn1`` /
``rgcn2`` (so state_dict keys ``aggregator.rgcn{1,2}.{weight,loop_weight}`` carry over),
``forward`` / ``predict_batch`` returning two ``PackedSequence`` (4h and 3h wide, sequences sorted by
history length, time-major), ``predict`` returning dense ``[len,4h]`` / ``[len,3h]`` tensors.

New (used by ``RENet.forward``): ``encode`` runs history batching -> 2 fused RGCN layers -> fused
read-out + GRU without ever materialising the padded/packed inputs.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.utils.rnn import PackedSequence

from . import _lib
from .rgcn import RGCNBlockLayer as RGCNLayer
from .utils import assemble_history_batch, global_rows, global_rows_of_batch


class _PackInputsFn(torch.autograd.Function):
    """X4/X3 in packed (time-major) order, Aggregator.py:139-165 without the Python loop."""

    @staticmethod
    def forward(ctx, H2, ent, rel, glob, hb, seq_s, seq_r, readout=None):
        L = _lib.lib()
        readout = hb.readout if readout is None else readout
        _lib.require_cuda(H2, ent, rel, glob)
        H2, ent, rel, glob = H2.contiguous(), ent.contiguous(), rel.contiguous(), glob.contiguous()
        h = H2.shape[1]
        X4 = torch.empty(hb.S, 4 * h, device=H2.device)
        X3 = torch.empty(hb.S, 3 * h, device=H2.device)
        rc = L.renet_pack_inputs(_lib.ptr(H2), _lib.ptr(readout), _lib.ptr(hb.row_glob), _lib.ptr(glob),
                                 _lib.ptr(ent), _lib.ptr(rel), _lib.ptr(hb.row_seq), _lib.ptr(seq_s),
                                 _lib.ptr(seq_r), _lib.ptr(hb.packed_row), _lib.ptr(X4), _lib.ptr(X3), hb.S, h,
                                 _lib.stream())
        _lib.check(rc, 'renet_pack_inputs')
        ctx.hb, ctx.seq_s, ctx.seq_r, ctx.readout = hb, seq_s, seq_r, readout
        ctx.shapes = (H2.shape, ent.shape, rel.shape, glob.shape)
        return X4, X3

    @staticmethod
    def backward(ctx, dX4, dX3):
        hb, h = ctx.hb, ctx.shapes[0][1]
        row = hb.packed_row.long()
        q = hb.row_seq.long()[row]
        dev = dX4.device
        dH2 = torch.zeros(ctx.shapes[0], device=dev).index_add_(0, ctx.readout.long()[row], dX4[:, :h] + dX3[:, :h])
        dent = torch.zeros(ctx.shapes[1], device=dev).index_add_(0, ctx.seq_s.long()[q], dX4[:, h:2 * h] + dX3[:, h:2 * h])
        drel = torch.zeros(ctx.shapes[2], device=dev).index_add_(0, ctx.seq_r.long()[q], dX4[:, 2 * h:3 * h])
        dglob = torch.zeros(ctx.shapes[3], device=dev).index_add_(0, hb.row_glob.long()[row], dX4[:, 3 * h:] + dX3[:, 2 * h:])
        return dH2, dent, drel, dglob, None, None, None, None


class RGCNAggregator(nn.Module):
    def __init__(self, h_dim, dropout, num_nodes, num_rels, num_bases, model, seq_len=10):
        super(RGCNAggregator, self).__init__()
        self.h_dim = h_dim
        self.dropout = nn.Dropout(dropout)
        self.seq_len = seq_len
        self.num_rels = num_rels
        self.num_nodes = num_nodes
        self.model = model
        self.rgcn1 = RGCNLayer(self.h_dim, self.h_dim, 2 * self.num_rels, num_bases,
                               activation=F.relu, self_loop=True, dropout=dropout)
        self.rgcn2 = RGCNLayer(self.h_dim, self.h_dim, 2 * self.num_rels, num_bases,
                               activation=None, self_loop=True, dropout=dropout)
        self._pack_token = _lib.new_pack_token()

    # ---------------------------------------------------------------------------------------------
    def _batch(self, s_hist, s, graph_dict, device, sort):
        from .hoststore import GraphStore, HistoryView, assemble_view, view_from_lists
        from .utils import HistoryBatch
        if isinstance(s_hist, HistoryBatch):         # already assembled and uploaded (hoststore.prefetch)
            if s_hist.graph is None:
                raise ValueError('RGCNAggregator: every history in the batch is empty '
                                 '(the reference fails on this input too, Aggregator.py:128-129,167)')
            return s_hist
        if isinstance(s_hist, HistoryView):          # flat stores + C++ batcher (renet_host_assemble_batch)
            if s_hist.total_length() == 0:
                raise ValueError('RGCNAggregator: every history in the batch is empty '
                                 '(the reference fails on this input too, Aggregator.py:128-129,167)')
            return assemble_view(s_hist, device, sort)
        total = 0
        for his in s_hist[0]:
            total += len(his)
        if total == 0:
            # the reference returns an unbound local here (Aggregator.py:128-129,167) and crashes
            raise ValueError('RGCNAggregator: every history in the batch is empty '
                             '(the reference fails on this input too, Aggregator.py:128-129,167)')
        s_host = s.detach().reshape(-1).cpu().numpy()
        if isinstance(graph_dict, GraphStore):
            # the reference's list inputs with a flattened graph store: flatten the batch on the fly and use the C++ /
            # device batcher (10 ms of host work per direction instead of the numpy path's 50-100 ms)
            return assemble_view(view_from_lists(s_hist[0], s_hist[1], s_host, graph_dict), device, sort)
        return assemble_history_batch(s_hist[0], s_hist[1], s_host, graph_dict, device, sort=sort)

    def aggregate(self, hb, ent_embeds, reverse):
        """The two RGCN layers over the batched history graph (Aggregator.py:136-139); the embedding lookup
        ndata['h'] = ent_embeds[id] (utils.py:239) is fused into layer 1.  Layer 2 runs on the read-out sub-graph only
        (Aggregator.py:140 keeps nothing but the read-out rows of its output): returns (H2c [S_cap, h], readout_c) with
        H2c[readout_c[i]] == the reference's embeds_mean[node_ids_graph][i]."""
        g = hb.graph
        H1 = self.rgcn1.apply_layer(g, ent_embeds, g.node_ent, reverse)
        sub = g.readout_sub(hb.readout, reverse)
        return self.rgcn2.apply_layer(sub, H1, None, reverse, loop_index=sub.uniq), sub.readout_c

    def _sorted_ids(self, hb, s, r, device):
        idx = hb.sample_order(device)
        s_tem, r_tem = s.reshape(-1)[idx], r.reshape(-1)[idx]
        Q = hb.num_seq
        return s_tem, r_tem, s_tem[:Q].to(torch.int32).contiguous(), r_tem[:Q].to(torch.int32).contiguous()

    def _packed(self, s_hist, s, r, ent_embeds, rel_embeds, graph_dict, global_emb, reverse, sort):
        dev = ent_embeds.device
        hb = self._batch(s_hist, s, graph_dict, dev, sort)
        H2, readout = self.aggregate(hb, ent_embeds, reverse)
        glob = global_rows(global_emb, hb.times, self.h_dim, dev)
        _, _, seq_s, seq_r = self._sorted_ids(hb, s, r, dev)
        X4, X3 = _PackInputsFn.apply(H2, ent_embeds, rel_embeds, glob, hb, seq_s, seq_r, readout)
        X4, X3 = self.dropout(X4), self.dropout(X3)                       # Aggregator.py:157-158
        bs = torch.from_numpy(hb.batch_sizes.astype(np.int64))
        return PackedSequence(X4, bs), PackedSequence(X3, bs), hb

    def forward(self, s_hist, s, r, ent_embeds, rel_embeds, graph_dict, global_emb, reverse):
        """Reference Aggregator.py:124-167."""
        p4, p3, _ = self._packed(s_hist, s, r, ent_embeds, rel_embeds, graph_dict, global_emb, reverse, True)
        return p4, p3

    def predict_batch(self, s_hist, s, r, ent_embeds, rel_embeds, graph_dict, global_emb, reverse):
        """Reference Aggregator.py:169-214 (unsorted twin)."""
        p4, p3, _ = self._packed(s_hist, s, r, ent_embeds, rel_embeds, graph_dict, global_emb, reverse, False)
        return p4, p3

    def predict(self, s_history, s, r, ent_embeds, rel_embeds, graph_dict, global_emb, reverse):
        """Reference Aggregator.py:218-237: one (s, r) history -> dense [len,4h], [len,3h]."""
        p4, p3, hb = self._packed(([s_history[0]], [s_history[1]]), s.view(-1, 1), r.view(-1, 1), ent_embeds,
                                  rel_embeds, graph_dict, global_emb, reverse, False)
        return p4.data, p3.data          # a single sequence: packed order == time order

    # ---------------------------------------------------------------------------------------------
    def encode(self, hist, s, r, ent_embeds, rel_embeds, graph_dict, global_emb, reverse, encoder, encoder_r, triplets=None):
        """history -> RGCN x2 -> fused read-out + both GRUs.  Returns (s_h, s_q, hb) with Q rows (non-empty histories,
        length-sorted), or already zero-padded to len(s) rows on the no-autograd path.  ``triplets`` (optional, the int64
        [B,3] batch s and r are columns of) lets that path build the sequence ids in one launch."""
        from .gru import fused_gru
        dev = ent_embeds.device
        hb = self._batch(hist, s, graph_dict, dev, True)
        # weights the tensor-core GEMM engine packs: unchanged weights (same addresses, same in-place versions) are packed
        # once and reused across calls -- both directions of a step, and every step in inference
        weights = [self.rgcn1.loop_weight, self.rgcn2.loop_weight, encoder.weight_ih_l0, encoder.weight_hh_l0,
                   encoder_r.weight_ih_l0, encoder_r.weight_hh_l0]
        with _lib.weight_generation(self._pack_token, weights):
            if not torch.is_grad_enabled() and not self.training:
                return self._encode_inference(hb, s, r, ent_embeds, rel_embeds, global_emb, reverse, encoder, encoder_r, triplets)
            H2, readout = self.aggregate(hb, ent_embeds, reverse)
            glob = global_rows_of_batch(global_emb, hb, self.h_dim, dev)
            _, _, seq_s, seq_r = self._sorted_ids(hb, s, r, dev)
            p_drop = self.dropout.p if self.training else 0.0          # Aggregator.py:157-158
            s_h, s_q = fused_gru(H2, ent_embeds, rel_embeds, glob, hb, seq_s, seq_r, encoder, encoder_r, readout=readout,
                                 p_drop=p_drop)
            return s_h, s_q, hb

    def _encode_inference(self, hb, s, r, ent_embeds, rel_embeds, global_emb, reverse, encoder, encoder_r, triplets=None):
        """No-autograd fast path: the whole direction (2 RGCN layers + read-out + both GRUs) is ONE C-ABI call
        (renet_encode_fwd), so the Python cost per direction is a handful of tensor ops instead of ~60.  Returns the GRU
        states zero-padded to len(s) rows (model.py:88,96)."""
        from .gru import _gru_params
        from .utils import _global_table
        L = _lib.lib()
        P = _lib.ptr
        dev = ent_embeds.device
        g, h = hb.graph, self.h_dim
        Q, B = hb.num_seq, s.numel()
        cg, gs = getattr(hb, 'comp_graph_dev', None), getattr(hb, 'graph_store', None)
        fast = (triplets is not None and cg is not None and gs is not None and triplets.dtype == torch.int64 and
                triplets.is_cuda and triplets.is_contiguous() and triplets.dim() == 2 and triplets.shape[1] >= 3)
        if fast:
            table, keys = _global_table(global_emb, h, dev)
            fast = len(keys) == len(gs.times) and (keys is gs.times or np.array_equal(keys, gs.times))
        if fast:
            # sequence ids and the read-out rows' global-table index in one launch (renet_prepare_sequences)
            ids = torch.empty(2 * Q + hb.S, dtype=torch.int32, device=dev)
            seq_s, seq_r, row_glob = ids[:Q], ids[Q:2 * Q], ids[2 * Q:]
            _lib.check(L.renet_prepare_sequences(P(triplets), triplets.shape[1], 2 if reverse else 0, P(hb.s_idx_dev), Q, P(cg), P(hb.row_glob),
                                                 hb.S, P(seq_s), P(seq_r), P(row_glob), _lib.stream()), 'renet_prepare_sequences')
            glob = table
        else:
            glob = global_rows_of_batch(global_emb, hb, h, dev)
            idx = hb.sample_order(dev)
            seq_s = s.reshape(-1)[idx][:Q].to(torch.int32)
            seq_r = r.reshape(-1)[idx][:Q].to(torch.int32)
            row_glob = hb.row_glob
        p4, p3 = _gru_params(encoder), _gru_params(encoder_r)
        rel = rel_embeds.contiguous()
        T = glob.shape[0]
        sub = g.readout_sub(hb.readout, reverse)       # layer 2 runs on the read-out sub-graph (Aggregator.py:140)
        H = torch.empty(g.N + hb.S, h, device=dev)     # H1 [N] | H2 compact [S]
        hn = torch.zeros(2, B, h, device=dev)          # rows >= Q stay zero: samples without history
        nbytes = int(L.renet_gru_workspace_bytes(hb.S, Q, T, h))
        ws = torch.empty(nbytes // 4 + 4, dtype=torch.float32, device=dev)
        bs = hb.batch_sizes
        l1, l2 = self.rgcn1, self.rgcn2
        hot = g.hot_rel(reverse)
        rc = L.renet_encode_fwd(P(ent_embeds), P(g.node_ent), P(g.row_ptr), P(g.col_src), P(g.col_type(reverse)),
                                P(g.norm), P(l1.weight), P(l1.loop_weight), P(l2.weight), P(l2.loop_weight), P(H),
                                P(H[g.N:]), g.N, g.E_launch, l1.weight.shape[0], P(hb.readout), P(row_glob), P(glob), P(rel),
                                P(seq_s), P(seq_r), P(g.seq_len_dev), P(hb.seq_start),
                                bs.ctypes.data_as(_lib.ctypes.c_void_p), len(bs), P(p4[0]), P(p4[1]), P(p4[2]), P(p4[3]),
                                P(p3[0]), P(p3[1]), P(p3[2]), P(p3[3]), P(hn[0]), P(hn[1]), hb.S, Q, T, h, l1.num_bases,
                                P(sub.uniq), P(sub.readout_c), P(sub.row_ptr), P(sub.col_src), P(sub.col_type(reverse)),
                                P(sub.norm), P(hot), 0 if hot is None else hot.numel(), P(ws), nbytes, _lib.stream())
        _lib.check(rc, 'renet_encode_fwd')
        return hn[0], hn[1], hb
