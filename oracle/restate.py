"""TEST INFRASTRUCTURE ONLY -- CPU restatement (numpy / torch-CPU fp32) of the RE-Net hot path.

This file travels to the GPU box (``/root/reference`` does not) and is what ``tests/ -m gpu``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs check and
time against.  It is never imported by the product package ``renet_b200``.

Pinning status: the reference has NO tests / golden vectors for this path (SURVEY.md section 4), and
the per-destination reduction lives in DGL 0.4.x (``dgl<0.5``, reference README.md:38), which is not
vendored.  Every function below is therefore pinned against OUTPUTS OF THE REFERENCE ITSELF, run
in the authoring container through ``oracle/ref_loader.py`` (unmodified reference modules over a
pure-torch DGL stand-in): see ``oracle/gen_golden.py`` -> ``tests/golden/*.npz`` and
``tests/test_oracle_vs_reference.py``.  At the DGL boundary the semantics come from DGL 0.4
documentation, i.e. "parity unpinned" by any reference-owned vector.

Each function cites the reference file:line it follows.
"""
from collections import defaultdict

import numpy as np
import torch


# --------------------------------------------------------------------------------------------------
# graph construction (input format definition)
# --------------------------------------------------------------------------------------------------
class PlainGraph:
    """DGL-free per-timestamp graph: what utils.get_big_graph (utils.py:68-87) produces."""

    def __init__(self, ids, src, dst, type_s, type_o):
        self.id = np.asarray(ids, dtype=np.int64)            # ndata['id']  [n]
        self.src = np.asarray(src, dtype=np.int64)           # local rows
        self.dst = np.asarray(dst, dtype=np.int64)
        self.type_s = np.asarray(type_s, dtype=np.int64)     # edata['type_s'] [e]
        self.type_o = np.asarray(type_o, dtype=np.int64)
        self.norm = comp_deg_norm(len(self.id), self.dst)    # ndata['norm'] [n]
        self.ids = {int(e): i for i, e in enumerate(self.id)}  # g.ids (utils.py:82-86)

    def number_of_nodes(self):
        return len(self.id)

    def number_of_edges(self):
        return len(self.src)


def comp_deg_norm(n, dst):
    """utils.py:89-93: norm = 1 / max(in_degree, 1), float32."""
    deg = np.bincount(np.asarray(dst, dtype=np.int64), minlength=n).astype(np.float32)
    deg[deg == 0] = 1.0
    return (np.float32(1.0) / deg).astype(np.float32)


def get_big_graph(triples, num_rels):
    """utils.py:68-87.  triples int [n,3] = (s, r, o) of ONE timestamp.

    nodes = sorted unique entities (np.unique, :70); edges = [s->o ..., o->s ...] (:74);
    type_s = [r..., r+R...] (:76), type_o = [r+R..., r...] (:75); duplicates kept.
    """
    triples = np.asarray(triples, dtype=np.int64)
    s, r, o = triples[:, 0], triples[:, 1], triples[:, 2]
    uniq_v, inv = np.unique(np.stack((s, o)), return_inverse=True)
    ls, lo = np.reshape(inv, (2, -1))
    src = np.concatenate((ls, lo))
    dst = np.concatenate((lo, ls))
    type_o = np.concatenate((r + num_rels, r))
    type_s = np.concatenate((r, r + num_rels))
    return PlainGraph(uniq_v, src, dst, type_s, type_o)


def build_graph_dict(quads, num_rels):
    """data/ICEWS18/get_history_graph.py:137-140: one graph per distinct timestamp."""
    quads = np.asarray(quads, dtype=np.int64)
    out = {}
    for t in np.unique(quads[:, 3]):
        out[int(t)] = get_big_graph(quads[quads[:, 3] == t][:, :3], num_rels)
    return out


def build_history(quads, num_e, history_len=10):
    """data/ICEWS18/get_history_graph.py:142-190 (train split).

    Per-entity rolling history: events of the current timestamp are cached and only become visible
    when the timestamp changes; keep the last ``history_len`` timestamps; each history entry is an
    int array [k,2] of (r, other-entity) plus its timestamp.  Returns
    (s_hist, s_hist_t, o_hist, o_hist_t), each a list over quads.
    The reference flushes every entity on a timestamp change (:147-169); flushing lazily the set
    of entities touched in the closing timestamp is the same thing.
    """
    quads = np.asarray(quads, dtype=np.int64)
    s_his = defaultdict(list); s_his_t = defaultdict(list)
    o_his = defaultdict(list); o_his_t = defaultdict(list)
    s_cache = defaultdict(list); o_cache = defaultdict(list)
    s_cache_t = {}; o_cache_t = {}
    S, ST, O, OT = [], [], [], []
    latest_t = 0

    def flush(cache, cache_t, his, his_t):
        for ee in sorted(cache.keys()):
            if len(cache[ee]) == 0:
                continue
            if len(his[ee]) >= history_len:
                his[ee].pop(0); his_t[ee].pop(0)
            his[ee].append(np.asarray(cache[ee], dtype=np.int64).reshape(-1, 2))
            his_t[ee].append(cache_t[ee])
        cache.clear(); cache_t.clear()

    for s, r, o, t in quads:
        s, r, o, t = int(s), int(r), int(o), int(t)
        if latest_t != t:
            flush(s_cache, s_cache_t, s_his, s_his_t)
            flush(o_cache, o_cache_t, o_his, o_his_t)
            latest_t = t
        S.append(list(s_his[s])); ST.append(list(s_his_t[s]))
        O.append(list(o_his[o])); OT.append(list(o_his_t[o]))
        s_cache[s].append([r, o]); s_cache_t[s] = t
        o_cache[o].append([r, s]); o_cache_t[o] = t
    return S, ST, O, OT


# --------------------------------------------------------------------------------------------------
# batched history-graph assembly
# --------------------------------------------------------------------------------------------------
def induced_subgraph(g, nodes):
    """utils.make_subgraph (utils.py:115-131) over DGL 0.4 ``subgraph``.

    ``nodes`` = iterable of ENTITY ids; local order = the given order.  Keeps every parallel edge
    whose two endpoints are selected, copies id/type_s/type_o, RECOMPUTES norm on the sub-graph
    (:126-127) and rebuilds ids (:129-130).
    """
    nodes = [int(x) for x in nodes]
    parent_rows = np.asarray([g.ids[e] for e in nodes], dtype=np.int64)
    new_id = np.full(g.number_of_nodes(), -1, dtype=np.int64)
    new_id[parent_rows] = np.arange(len(parent_rows))
    keep = (new_id[g.src] >= 0) & (new_id[g.dst] >= 0)
    return PlainGraph(g.id[parent_rows], new_id[g.src[keep]], new_id[g.dst[keep]],
                      g.type_s[keep], g.type_o[keep])


class BatchedHistory:
    """Everything utils.get_sorted_s_r_embed_rgcn (utils.py:209-244) hands to the aggregator."""
    pass


def assemble_batch(hist, hist_t, s, sort=True, node_order=None):
    """utils.py:209-244 (sort=True) / :246-283 (sort=False), without the embedding lookups.

    hist: list[B] of list[<=L] of int arrays [k,2]; hist_t: list[B] of list of timestamps;
    s: int array [B].  Sorting by history length uses a STABLE descending sort; the reference's
    torch sort (model.py:81) leaves tie order unspecified and the loss is invariant to it.
    ``node_order(t, set) -> list`` fixes the node order inside each sub-graph (default: sorted).
    """
    B = len(hist)
    lens = np.asarray([len(h) for h in hist], dtype=np.int64)
    idx = np.argsort(-lens, kind='stable') if sort else np.arange(B)
    if sort:
        nnz = int((lens > 0).sum())
    else:
        # utils.py:253-255: the unsorted twin truncates at the COUNT of non-empty histories
        nnz = int((lens > 0).sum())
    out = BatchedHistory()
    out.s_idx = idx
    out.seq_len = lens[idx][:nnz]
    hs = [hist[i] for i in idx[:nnz]]
    hts = [hist_t[i] for i in idx[:nnz]]
    s_tem = np.asarray(s, dtype=np.int64)[idx]
    # utils.py:149-156
    neighs_t = {}
    for i, (h, ht) in enumerate(zip(hs, hts)):
        for neighs, t in zip(h, ht):
            st = neighs_t.setdefault(int(t), set())
            st.update(int(x) for x in np.asarray(neighs)[:, 1])
            st.add(int(s_tem[i]))
    out.times = list(neighs_t.keys())           # dict insertion order, as utils.py:162
    out.node_sets = neighs_t
    out.row_time = [int(t) for ht in hts for t in ht]       # timestamp of every read-out row
    out.row_seq = [i for i, ht in enumerate(hts) for _ in ht]
    out.s_tem = s_tem
    out.node_order = node_order or (lambda t, st: sorted(st))
    return out


def batch_graphs(bh, graph_dict):
    """utils.py:158-181 + dgl.batch (:238): disjoint union with node offsets; read-out rows."""
    subs, start, off = [], {}, 0
    for t in bh.times:
        sg = induced_subgraph(graph_dict[t], bh.node_order(t, bh.node_sets[t]))
        sg.start_id = off
        start[t] = (len(subs), off)
        off += sg.number_of_nodes()
        subs.append(sg)
    g = BatchedHistory()
    g.num_nodes = off
    g.id = np.concatenate([x.id for x in subs]) if subs else np.zeros(0, np.int64)
    g.norm = np.concatenate([x.norm for x in subs]) if subs else np.zeros(0, np.float32)
    g.src = np.concatenate([x.src + x.start_id for x in subs]) if subs else np.zeros(0, np.int64)
    g.dst = np.concatenate([x.dst + x.start_id for x in subs]) if subs else np.zeros(0, np.int64)
    g.type_s = np.concatenate([x.type_s for x in subs]) if subs else np.zeros(0, np.int64)
    g.type_o = np.concatenate([x.type_o for x in subs]) if subs else np.zeros(0, np.int64)
    g.comp_sizes = [x.number_of_nodes() for x in subs]
    # utils.py:172-181: read-out row = ids[s] + start_id
    rows = []
    for i, t in zip(bh.row_seq, bh.row_time):
        k, o = start[t]
        rows.append(subs[k].ids[int(bh.s_tem[i])] + o)
    g.readout = np.asarray(rows, dtype=np.int64)
    return g


# --------------------------------------------------------------------------------------------------
# RGCN block layer
# --------------------------------------------------------------------------------------------------
# rgcn_block_layer gathers W[etype] for at most this many edges at once: a whole-graph batch of 3.5 M edges would need 11 GB
# in float64
EDGE_CHUNK = 1 << 18


def rgcn_block_layer(H, W, Wloop, src, dst, etype, norm, relu, num_bases):
    """Closed form of RGCNLayer.forward + RGCNBlockLayer (RGCN.py:33-51, 79-94), dropout off:

        out = act( norm * sum_{e: dst(e)=v} blockdiag(W[etype_e]) . H[src_e]  +  H @ Wloop )

    H [N,din] fp32, W [R2, nb*si*so], Wloop [din,dout] or None, src/dst/etype int64 [E],
    norm [N] fp32.  torch-CPU fp32; differentiable (used for backward parity too).
    """
    N, din = H.shape
    nb = num_bases
    si = din // nb
    so = W.shape[1] // (nb * si)
    dout = nb * so
    if src.numel() > 0:
        agg = torch.zeros(N, dout, dtype=H.dtype, device=H.device)
        for a in range(0, src.numel(), EDGE_CHUNK):            # the same adds in the same order, a chunk of edges at a time
            e = slice(a, a + EDGE_CHUNK)
            w = W[etype[e]].view(-1, nb, si, so)               # RGCN.py:81-85
            x = H[src[e]].view(-1, nb, si)                     # RGCN.py:86
            msg = torch.einsum('ebi,ebij->ebj', x, w).reshape(-1, dout)   # RGCN.py:87
            agg = agg.index_add(0, dst[e], msg)                # fn.sum, RGCN.py:91
    else:
        agg = H if din == dout else torch.zeros(N, dout, dtype=H.dtype, device=H.device)  # DGL 0.4: reduce skipped
    out = agg * norm.view(-1, 1)                               # RGCN.py:93-94
    if Wloop is not None:
        out = out + H @ Wloop                                  # RGCN.py:35,45-46
    return torch.relu(out) if relu else out                    # RGCN.py:47-48


def rgcn_block_layer_ref_ops(H, W, Wloop, src, dst, etype, norm, relu, num_bases):
    """Same result, but with the reference's OWN op sequence (index_select -> view(-1,si,so) ->
    bmm of E*nb tiny matrices -> index_add), RGCN.py:79-88.  This is the shape of work the reference
    puts on the CPU and is what the ``cpu_baseline`` leg of bench.py times."""
    N, din = H.shape
    nb = num_bases
    si = din // nb
    so = W.shape[1] // (nb * si)
    weight = W.index_select(0, etype).view(-1, si, so)
    node = H[src].view(-1, 1, si)
    msg = torch.bmm(node, weight).view(-1, nb * so)
    agg = torch.zeros(N, nb * so, dtype=H.dtype).index_add_(0, dst, msg)
    out = agg * norm.view(-1, 1)
    if Wloop is not None:
        out = out + torch.mm(H, Wloop)
    return torch.relu(out) if relu else out


# --------------------------------------------------------------------------------------------------
# read-out, concat, GRU
# --------------------------------------------------------------------------------------------------
def packed_inputs(H2, readout, seq_len, s_tem, r_tem, ent, rel, glob_rows):
    """Aggregator.py:139-165 (dropout off): rows of X4 = [H2[readout] | ent[s] | rel[r] | glob[t]],
    X3 = [H2[readout] | ent[s] | glob[t]], returned sequence-major [S,4h],[S,3h] plus the packed
    (time-major) permutation that pack_padded_sequence(batch_first=True) applies, and batch_sizes."""
    rows = H2[readout]
    seq_of_row = torch.repeat_interleave(torch.arange(len(seq_len)), torch.as_tensor(seq_len)).to(s_tem.device)
    e = ent[s_tem[seq_of_row]]
    r = rel[r_tem[seq_of_row]]
    X4 = torch.cat((rows, e, r, glob_rows), dim=1)
    X3 = torch.cat((rows, e, glob_rows), dim=1)
    perm, batch_sizes = packed_order(seq_len)
    return X4, X3, perm, batch_sizes


def packed_order(seq_len):
    """Row permutation of pack_padded_sequence for lengths sorted descending: time-major."""
    seq_len = [int(x) for x in seq_len]
    starts = np.concatenate(([0], np.cumsum(seq_len)[:-1])) if seq_len else np.zeros(0, np.int64)
    perm, batch_sizes = [], []
    for t in range(max(seq_len) if seq_len else 0):
        n = sum(1 for l in seq_len if l > t)
        batch_sizes.append(n)
        perm.extend(int(starts[i]) + t for i in range(n))
    return np.asarray(perm, dtype=np.int64), np.asarray(batch_sizes, dtype=np.int64)


def gru_final_hidden(X, seq_len, w_ih, w_hh, b_ih, b_hh):
    """nn.GRU(1 layer, h0=0) final hidden per sequence (model.py:86,94), gate order (r,z,n):
        r = sig(W_ir x + b_ir + W_hr h + b_hr);  z = sig(W_iz x + b_iz + W_hz h + b_hz)
        n = tanh(W_in x + b_in + r * (W_hn h + b_hn));  h' = (1 - z) * n + z * h
    X [S,in] sequence-major rows (sequence i owns rows start_i .. start_i+len_i)."""
    Q = len(seq_len)
    hdim = w_hh.shape[1]
    h = torch.zeros(Q, hdim, dtype=X.dtype)
    starts = np.concatenate(([0], np.cumsum(seq_len)[:-1])).astype(np.int64)
    gi_all = X @ w_ih.t() + b_ih
    outs = []
    for q in range(Q):
        hq = torch.zeros(hdim, dtype=X.dtype)
        for t in range(int(seq_len[q])):
            gi = gi_all[starts[q] + t]
            gh = w_hh @ hq + b_hh
            r = torch.sigmoid(gi[:hdim] + gh[:hdim])
            z = torch.sigmoid(gi[hdim:2 * hdim] + gh[hdim:2 * hdim])
            n = torch.tanh(gi[2 * hdim:] + r * gh[2 * hdim:])
            hq = (1 - z) * n + z * hq
        outs.append(hq)
    return torch.stack(outs) if outs else h


def gru_final_hidden_batched(X, seq_len, w_ih, w_hh, b_ih, b_hh):
    """Same as gru_final_hidden, vectorised over sequences per time step (lengths sorted desc).  Runs in X's dtype on X's
    device."""
    seq_len = np.asarray(seq_len, dtype=np.int64)
    Q = len(seq_len)
    hdim = w_hh.shape[1]
    starts = torch.as_tensor(np.concatenate(([0], np.cumsum(seq_len)[:-1])).astype(np.int64), device=X.device)
    gi_all = X @ w_ih.t() + b_ih
    h = torch.zeros(Q, hdim, dtype=X.dtype, device=X.device)
    for t in range(int(seq_len.max()) if Q else 0):
        n_act = int((seq_len > t).sum())
        gi = gi_all[starts[:n_act] + t]
        hp = h[:n_act]
        gh = hp @ w_hh.t() + b_hh
        r = torch.sigmoid(gi[:, :hdim] + gh[:, :hdim])
        z = torch.sigmoid(gi[:, hdim:2 * hdim] + gh[:, hdim:2 * hdim])
        n = torch.tanh(gi[:, 2 * hdim:] + r * gh[:, 2 * hdim:])
        h = torch.cat(((1 - z) * n + z * hp, h[n_act:]), dim=0)
    return h


# --------------------------------------------------------------------------------------------------
# whole forward of one direction (model.py:64-104), dropout off
# --------------------------------------------------------------------------------------------------
def renet_forward(params, triplets, hist, hist_t, graph_dict, global_emb, subject, num_rels,
                  num_bases=100, node_order=None):
    """params: dict of torch fp32 tensors keyed like RENet.state_dict().  Returns dict with loss,
    s_h, s_q, packed inputs, H1, H2 and the batched graph (for kernel-level comparisons)."""
    P = params
    R = num_rels
    tr = np.asarray(triplets, dtype=np.int64)
    if subject:                                               # model.py:65-71
        rel = P['rel_embeds'][:R]; s, r, o = tr[:, 0], tr[:, 1], tr[:, 2]; reverse = False
    else:                                                     # model.py:72-78
        rel = P['rel_embeds'][R:]; o, r, s = tr[:, 0], tr[:, 1], tr[:, 2]; reverse = True
    ent = P['ent_embeds']
    bh = assemble_batch(hist, hist_t, s, sort=True, node_order=node_order)
    g = batch_graphs(bh, graph_dict)
    idx = bh.s_idx
    s_tem, r_tem, o_tem = torch.as_tensor(s[idx]), torch.as_tensor(r[idx]), torch.as_tensor(o[idx])
    et = torch.as_tensor(g.type_o if reverse else g.type_s)  # RGCN.py:80-85
    src, dst = torch.as_tensor(g.src), torch.as_tensor(g.dst)
    norm = torch.as_tensor(g.norm)
    H0 = ent[torch.as_tensor(g.id)]                           # utils.py:239
    H1 = rgcn_block_layer(H0, P['aggregator.rgcn1.weight'], P['aggregator.rgcn1.loop_weight'],
                          src, dst, et, norm, True, num_bases)
    H2 = rgcn_block_layer(H1, P['aggregator.rgcn2.weight'], P['aggregator.rgcn2.loop_weight'],
                          src, dst, et, norm, False, num_bases)
    glob = torch.stack([global_emb[t].view(-1) for t in bh.row_time])    # utils.py:224-225
    X4, X3, perm, bs = packed_inputs(H2, torch.as_tensor(g.readout), bh.seq_len, s_tem, r_tem,
                                     ent, rel, glob)
    s_h = gru_final_hidden_batched(X4, bh.seq_len, P['encoder.weight_ih_l0'], P['encoder.weight_hh_l0'],
                                   P['encoder.bias_ih_l0'], P['encoder.bias_hh_l0'])
    s_q = gru_final_hidden_batched(X3, bh.seq_len, P['encoder_r.weight_ih_l0'], P['encoder_r.weight_hh_l0'],
                                   P['encoder_r.bias_ih_l0'], P['encoder_r.bias_hh_l0'])
    B, h = len(s), ent.shape[1]
    s_h_pad = torch.cat((s_h, s_h.new_zeros(B - len(s_h), h)), dim=0)   # model.py:88
    s_q_pad = torch.cat((s_q, s_q.new_zeros(B - len(s_q), h)), dim=0)   # model.py:96
    ob_pred = torch.cat((ent[s_tem], s_h_pad, rel[r_tem]), dim=1) @ P['linear.weight'].t() + P['linear.bias']
    loss_sub = torch.nn.functional.cross_entropy(ob_pred, o_tem)         # model.py:89-91
    ob_pred_r = torch.cat((ent[s_tem], s_q_pad), dim=1) @ P['linear_r.weight'].t() + P['linear_r.bias']
    loss_sub_r = torch.nn.functional.cross_entropy(ob_pred_r, r_tem)     # model.py:98-100
    return dict(loss=loss_sub + 0.1 * loss_sub_r, s_h=s_h, s_q=s_q, X4=X4, X3=X3, perm=perm,
                batch_sizes=bs, H0=H0, H1=H1, H2=H2, graph=g, batch=bh, etype=et)


# --------------------------------------------------------------------------------------------------
# global model (global_model.py, Aggregator.RGCNAggregator_global), dropout off
# --------------------------------------------------------------------------------------------------
def global_windows(t_list, times, seq_len=10):
    """Aggregator.py:28-45: t_list sorted descending; zeros (the first timestamp: no past) are dropped; each remaining t
    owns the <= seq_len graph timestamps before it."""
    time_unit = times[1] - times[0]
    out = []
    for tim in t_list:
        if int(tim) == 0:
            continue
        length = int(tim // time_unit)
        out.append(list(times[length - seq_len:length]) if seq_len <= length else list(times[:length]))
    return out


def global_pooled(params, window_times, graph_dict, reverse, maxpool, num_bases=100):
    """Aggregator.py:53-62 / 96-105: dgl.batch of WHOLE graphs, two block layers, max / mean over each graph's nodes."""
    P = params
    dev = P['ent_embeds'].device
    gs = [graph_dict[int(t)] for t in window_times]
    off = np.concatenate(([0], np.cumsum([g.number_of_nodes() for g in gs]))).astype(np.int64)
    src = torch.as_tensor(np.concatenate([g.src + o for g, o in zip(gs, off[:-1])]), device=dev)
    dst = torch.as_tensor(np.concatenate([g.dst + o for g, o in zip(gs, off[:-1])]), device=dev)
    et = torch.as_tensor(np.concatenate([g.type_o if reverse else g.type_s for g in gs]), device=dev)
    norm = torch.as_tensor(np.concatenate([g.norm for g in gs]), device=dev)
    H0 = P['ent_embeds'][torch.as_tensor(np.concatenate([g.id for g in gs]), device=dev)]
    H1 = rgcn_block_layer(H0, P['aggregator.rgcn1.weight'], P['aggregator.rgcn1.loop_weight'], src, dst, et, norm, True,
                          num_bases)
    H2 = rgcn_block_layer(H1, P['aggregator.rgcn2.weight'], P['aggregator.rgcn2.loop_weight'], src, dst, et, norm, False,
                          num_bases)
    rows = []
    for a, b in zip(off[:-1], off[1:]):
        rows.append(H2[a:b].max(dim=0).values if maxpool == 1 else H2[a:b].mean(dim=0))
    return torch.stack(rows)


def soft_cross_entropy(pred, soft_targets):
    """utils.py:287-290."""
    logp = torch.nn.functional.log_softmax(pred.double(), dim=1)
    return torch.mean(torch.sum(-soft_targets.double() * logp, 1))


def global_forward(params, t_list, true_prob_s, true_prob_o, graph_dict, subject, maxpool=1, seq_len=10, num_bases=100):
    """RENet_global.forward (global_model.py:35-55): loss of one direction for a batch of timestamps.  Runs on the device
    of ``params``."""
    P = params
    dev = P['ent_embeds'].device
    reverse = not subject
    lin = 'linear_s' if subject else 'linear_o'
    true_prob = torch.as_tensor(true_prob_o if subject else true_prob_s, device=dev)
    t_host = np.asarray(t_list, dtype=np.int64)
    idx = np.argsort(-t_host, kind='stable')                                    # global_model.py:45
    times = list(graph_dict.keys())
    windows = global_windows(t_host[idx], times, seq_len)
    uniq = sorted({int(t) for w in windows for t in w})                          # Aggregator.py:47
    pos = {t: i for i, t in enumerate(uniq)}
    info = global_pooled(P, uniq, graph_dict, reverse, maxpool, num_bases)
    X = info[torch.as_tensor([pos[int(t)] for w in windows for t in w], dtype=torch.long, device=dev)]
    lens = [len(w) for w in windows]
    s_q = gru_final_hidden_batched(X, lens, P['encoder_global.weight_ih_l0'], P['encoder_global.weight_hh_l0'],
                                   P['encoder_global.bias_ih_l0'], P['encoder_global.bias_hh_l0'])
    s_q = torch.cat((s_q, s_q.new_zeros(len(t_host) - len(s_q), s_q.shape[1])), dim=0)    # global_model.py:51
    pred = s_q @ P[lin + '.weight'].t() + P[lin + '.bias']
    return soft_cross_entropy(pred, true_prob[torch.as_tensor(idx, device=dev)])


def global_predict(params, t, graph_dict, subject=True, maxpool=1, seq_len=10, num_bases=100):
    """RENet_global.predict (global_model.py:77-89): (s_q [h], logits [in_dim]) from the graphs before time t."""
    P = params
    times = list(graph_dict.keys())
    k = sum(1 for tt in times if tt < t)                                         # Aggregator.py:78-82 (times ascend)
    window = times[k - seq_len:k] if seq_len <= k else times[:k]
    X = global_pooled(P, window, graph_dict, not subject, maxpool, num_bases)
    s_q = gru_final_hidden_batched(X, [len(window)], P['encoder_global.weight_ih_l0'], P['encoder_global.weight_hh_l0'],
                                   P['encoder_global.bias_ih_l0'], P['encoder_global.bias_hh_l0'])[0]
    lin = 'linear_s' if subject else 'linear_o'
    return s_q, P[lin + '.weight'] @ s_q + P[lin + '.bias']
