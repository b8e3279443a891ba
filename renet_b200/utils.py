"""Host-side batching of history graphs: the contract of reference utils.py:149-181, 209-283.

Same function names and return tuple as the reference (``get_sorted_s_r_embed_rgcn`` /
``get_s_r_embed_rgcn``) so call sites and tests read alike, but implemented on flat numpy arrays:
one pass collects (timestamp, entity) pairs of the whole batch, ``np.unique`` on a combined key
yields every per-timestamp node set at once, the induced sub-graphs are array masks over
destination-sorted per-timestamp edge lists (so the batched graph is born in CSR form, no sort), and
everything reaches the GPU in two pinned copies.  Nothing here touches ``.item()`` per element or
does per-row device copies (the reference does S of them, utils.py:225).
"""
import operator

import numpy as np
import torch

from .graph import BatchedHistoryGraph, HistoryGraph, as_history_graph, get_big_graph  # noqa: F401


class HistoryBatch:
    """Everything the aggregator needs for one direction of one batch."""
    __slots__ = ('s_idx', 'seq_len', 'num_seq', 'times', 'graph', 'readout', 'readout_host', 'row_glob',
                 'row_seq', 'seq_start', 'packed_row', 'batch_sizes', 'S', 'h2d_bytes', 's_idx_dev', 'comp_graph_dev',
                 'graph_store')

    def sample_order(self, device):
        """device int64 index of the samples in processing order (history length descending)."""
        dev_idx = getattr(self, 's_idx_dev', None)
        if dev_idx is not None:
            return dev_idx.long()
        return torch.from_numpy(self.s_idx).to(device)


def _history_order(hist_len, sort):
    hist_len = np.asarray(hist_len, dtype=np.int64)
    if sort:
        # reference: torch sort descending (model.py:81, utils.py:213); ties are unspecified there,
        # stable here.  The loss is invariant to the order among equal lengths.
        s_idx = np.argsort(-hist_len, kind='stable')
    else:
        s_idx = np.arange(len(hist_len))          # utils.py:251
    nnz = int(np.count_nonzero(hist_len))         # utils.py:214 / :253
    return s_idx, hist_len[s_idx][:nnz]


def assemble_history_batch(s_hist, s_hist_t, s_host, graph_dict, device, sort=True):
    """Core of utils.py:209-244: returns a HistoryBatch (graph already on ``device``)."""
    return upload_history_batch(assemble_history_batch_host(s_hist, s_hist_t, s_host, graph_dict, sort), device)


def assemble_history_batch_host(s_hist, s_hist_t, s_host, graph_dict, sort=True):
    """Host half of the batching: pure numpy, returns a HistoryBatch whose ``graph`` is a dict of
    host arrays (node_ent, norm, row_ptr, col_src, col_type_s, col_type_o, comp_sizes)."""
    s_idx, seq_len = _history_order([len(h) for h in s_hist], sort)
    Q = len(seq_len)
    hb = HistoryBatch()
    hb.s_idx, hb.seq_len, hb.num_seq = s_idx, seq_len, Q
    S = int(seq_len.sum())
    hb.S = S
    if S == 0:
        hb.graph = None
        return hb
    s_tem = np.asarray(s_host, dtype=np.int64)[s_idx]

    # ---- flatten the histories (utils.py:149-156) --------------------------------------------------
    ent_chunks, chunk_len, row_t = [], np.empty(S, dtype=np.int64), np.empty(S, dtype=np.int64)
    k = 0
    for i in range(Q):
        hist, hist_t = s_hist[s_idx[i]], s_hist_t[s_idx[i]]
        for neighs, t in zip(hist, hist_t):
            ent_chunks.append(neighs[:, 1])
            chunk_len[k] = len(neighs)
            row_t[k] = t
            k += 1
    row_seq = np.repeat(np.arange(Q, dtype=np.int64), seq_len)
    row_s = s_tem[row_seq]
    # timestamps in first-appearance order (dict insertion order in utils.py:158-170)
    uniq_t, first, t_idx_of_row = np.unique(row_t, return_index=True, return_inverse=True)
    order = np.argsort(first, kind='stable')
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    times = uniq_t[order]
    row_comp = rank[t_idx_of_row]                       # component index of every read-out row
    G = len(times)

    graphs = [as_history_graph(graph_dict[int(t)]) for t in times]
    M = int(max(int(g.node_id[-1]) for g in graphs)) + 1   # entity-id bound for the combined key
    neigh_ent = np.concatenate(ent_chunks).astype(np.int64) if ent_chunks else np.zeros(0, np.int64)
    neigh_comp = np.repeat(row_comp, chunk_len)
    keys = np.concatenate((neigh_comp * M + neigh_ent, row_comp * M + row_s))
    node_key = np.unique(keys)                          # sorted: by component, then entity id
    node_comp = node_key // M
    node_ent = node_key - node_comp * M
    comp_sizes = np.bincount(node_comp, minlength=G)
    comp_start = np.concatenate(([0], np.cumsum(comp_sizes)))
    readout = np.searchsorted(node_key, row_comp * M + row_s)      # utils.py:172-181

    # ---- induced sub-graphs (utils.make_subgraph, utils.py:115-131), already destination-sorted -----
    srcs, dsts, tss, tos = [], [], [], []
    for c in range(G):
        g = graphs[c]
        lo, hi = comp_start[c], comp_start[c + 1]
        rows = g.rows_of(node_ent[lo:hi])
        new_id = np.full(g.number_of_nodes(), -1, dtype=np.int64)
        new_id[rows] = np.arange(lo, hi)
        ns, nd = new_id[g.src], new_id[g.dst]
        keep = (ns >= 0) & (nd >= 0)
        srcs.append(ns[keep]); dsts.append(nd[keep]); tss.append(g.type_s[keep]); tos.append(g.type_o[keep])
        if not g._sorted:   # adapted graphs whose ids are not ascending: local dst order may be permuted
            o = np.argsort(dsts[-1], kind='stable')
            srcs[-1], dsts[-1], tss[-1], tos[-1] = srcs[-1][o], dsts[-1][o], tss[-1][o], tos[-1][o]
    src = np.concatenate(srcs); dst = np.concatenate(dsts)
    N = int(comp_start[-1])
    indeg = np.bincount(dst, minlength=N)
    row_ptr = np.concatenate(([0], np.cumsum(indeg)))
    deg = indeg.astype(np.float32)
    deg[deg == 0] = 1.0
    norm = (np.float32(1.0) / deg).astype(np.float32)              # recomputed per sub-graph, utils.py:126-127

    hb.times = times
    type_s, type_o = np.concatenate(tss), np.concatenate(tos)
    hb.graph = dict(node_ent=node_ent, norm=norm, row_ptr=row_ptr, col_src=src, col_type_s=type_s,
                    col_type_o=type_o, comp_sizes=comp_sizes)
    # ---- sequence bookkeeping (pack_padded_sequence order, Aggregator.py:160-165) ------------------
    seq_start = np.concatenate(([0], np.cumsum(seq_len)[:-1]))
    max_len = int(seq_len[0]) if sort else int(seq_len.max())
    batch_sizes = np.asarray([int(np.count_nonzero(seq_len > t)) for t in range(max_len)], dtype=np.int32)
    packed_row = np.concatenate([seq_start[:batch_sizes[t]] + t for t in range(max_len)])
    hb.seq_len = seq_len
    hb.batch_sizes = batch_sizes
    hb.readout_host = readout
    hb.readout = (readout, row_comp, row_seq, seq_start, seq_len, packed_row)     # host arrays until uploaded
    return hb


def upload_history_batch(hb, device):
    """Device half: two pinned host->device copies (graph structure, sequence bookkeeping)."""
    if hb.graph is None:
        return hb
    g = hb.graph
    S, Q = hb.S, hb.num_seq
    hb.graph = BatchedHistoryGraph(g['node_ent'], g['norm'], g['row_ptr'], g['col_src'], g['col_type_s'],
                                   g['col_type_o'], device)
    i32 = np.concatenate(hb.readout).astype(np.int32)
    dev = torch.from_numpy(i32).pin_memory().to(device, non_blocking=True)
    o = 0
    hb.readout = dev[o:o + S]; o += S
    hb.row_glob = dev[o:o + S]; o += S
    hb.row_seq = dev[o:o + S]; o += S
    hb.seq_start = dev[o:o + Q]; o += Q
    seq_len_dev = dev[o:o + Q]; o += Q
    hb.packed_row = dev[o:o + S]
    hb.h2d_bytes = hb.graph.h2d_bytes + i32.nbytes
    hb.graph.seq_len_dev = seq_len_dev
    return hb


_GLOB_CACHE = {}


def global_rows_of_batch(global_emb, hb, h, device):
    """global_rows for a HistoryBatch; when the batch came from the C++ batcher its component -> graph index is
    already on the device and the table is indexed without any host->device copy."""
    cg = getattr(hb, 'comp_graph_dev', None)
    gs = getattr(hb, 'graph_store', None)
    if cg is not None and gs is not None:
        table, keys = _global_table(global_emb, h, device)
        if len(keys) == len(gs.times) and (keys is gs.times or np.array_equal(keys, gs.times)):
            return table[cg.long()]
    return global_rows(global_emb, hb.times, h, device)


def _global_table(global_emb, h, device):
    """Dense [T,h] device table of the dict, cached per dict object.  The cache is dropped when the dict grows OR when
    any value object is replaced (the test-time roll-over overwrites global_emb[latest_time], model.py:302-303)."""
    key = id(global_emb)
    hit = _GLOB_CACHE.get(key)
    vals = list(global_emb.values())
    if (hit is None or hit[0] is not global_emb or len(hit[1]) != len(vals) or hit[3].device != torch.device(device)
            or not all(map(operator.is_, vals, hit[1]))):
        keys = np.asarray(sorted(int(t) for t in global_emb.keys()), dtype=np.int64)
        table = torch.stack([global_emb[int(t)].reshape(-1).to(device=device, dtype=torch.float32) for t in keys])   # entries may live on different devices
        hit = (global_emb, vals, keys, table.view(len(keys), h))
        _GLOB_CACHE.clear()
        _GLOB_CACHE[key] = hit
    return hit[3], hit[2]


def global_rows(global_emb, times, h, device):
    """[T,h] matrix of global_emb[t] for the batch's distinct timestamps.  The reference gathers one row per
    read-out row with a .cpu() each (utils.py:224-225); here the dict is turned into a dense device table
    once (cached per dict object) and a batch is one index_select."""
    table, keys = _global_table(global_emb, h, device)
    times = np.asarray(times, dtype=np.int64)
    idx = np.searchsorted(keys, times)
    bad = (idx >= len(keys)) | (keys[np.minimum(idx, len(keys) - 1)] != times)
    if np.any(bad):           # the reference indexes the dict and raises KeyError (utils.py:225)
        raise KeyError(int(times[np.flatnonzero(bad)[0]]))
    return table[torch.from_numpy(idx).to(device)]


def _wrap(hb, s, r, ent_embeds, global_emb):
    if hb.graph is None:
        return None, None, None, None, None, None
    dev = ent_embeds.device
    idx = torch.from_numpy(hb.s_idx).to(dev)
    g = hb.graph
    g.h_table, g.h_index = ent_embeds, g.node_ent       # ndata['h'] = ent_embeds[id]  (utils.py:239), lazily
    g.ndata['h'] = ent_embeds[g.node_ent.long()]
    glob = global_rows(global_emb, hb.times, ent_embeds.shape[1], dev)
    return (torch.from_numpy(hb.seq_len).to(dev), s[idx], r[idx], g, hb.readout_host.tolist(),
            glob[hb.row_glob.long()])


def get_sorted_s_r_embed_rgcn(s_hist_data, s, r, ent_embeds, graph_dict, global_emb):
    """Reference utils.py:209-244, same return tuple:
    (s_len_non_zero, s_tem, r_tem, batched_graph, node_ids_graph, global_emb_list)."""
    hb = assemble_history_batch(s_hist_data[0], s_hist_data[1], s.detach().cpu().numpy(), graph_dict,
                                ent_embeds.device, sort=True)
    return _wrap(hb, s, r, ent_embeds, global_emb)


def get_s_r_embed_rgcn(s_hist_data, s, r, ent_embeds, graph_dict, global_emb):
    """Reference utils.py:246-283 (unsorted twin used at inference)."""
    hb = assemble_history_batch(s_hist_data[0], s_hist_data[1], s.detach().view(-1).cpu().numpy(), graph_dict,
                                ent_embeds.device, sort=False)
    return _wrap(hb, s.view(-1), r.view(-1), ent_embeds, global_emb)
