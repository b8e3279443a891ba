"""Flat host-side stores + the C++ batcher (renet_host_assemble_batch): the fast path of
reference utils.get_sorted_s_r_embed_rgcn (utils.py:209-244).

The reference hands `RENet.forward` Python lists (`s_hist`: list[B] of list[<=10] of int arrays [k,2]) and a
dict of per-timestamp graphs, and re-walks them in Python for every batch.  Here both are flattened ONCE:

    gs = GraphStore(graph_dict)                       # all timestamps' graphs, CSR-ready
    hs = HistoryStore(s_hist_all, s_hist_t_all, subjects_all, gs)   # the training set's histories
    view = hs.select(sample_indices)                  # what a batch is: just indices

and ``model(triplets, view_s, view_o, gs, subject=...)`` assembles the batched history graph in C++ in a few
milliseconds, writes it into a pinned staging buffer and ships it to the GPU in one copy.  The list-based
API keeps working (numpy path in utils.py); both produce identical batches (tests/test_host_batching.py).
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .graph import BatchedHistoryGraph, PendingCount, _Frame, as_history_graph
from .utils import HistoryBatch

MAX_LEN = 16
N_HOT = 40          # relation rows renet_rgcn_gather_comp keeps in shared memory (kHotRel)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class GraphStore:
    """All per-timestamp graphs of a graph_dict, concatenated (nodes ascending by entity id, edges sorted by
    destination).  Quacks like the dict for the rest of the code (``store[t]``, ``in``, ``keys()``)."""

    def __init__(self, graph_dict):
        self.graph_dict = graph_dict
        self.times = np.asarray(sorted(int(t) for t in graph_dict.keys()), dtype=np.int64)
        self.index_of = {int(t): i for i, t in enumerate(self.times)}
        graphs = [as_history_graph(graph_dict[int(t)]) for t in self.times]
        for g in graphs:
            if not g._sorted:
                raise ValueError('GraphStore needs graphs whose node ids ascend (utils.get_big_graph order)')
        self.node_off = np.concatenate(([0], np.cumsum([g.number_of_nodes() for g in graphs]))).astype(np.int64)
        self.edge_off = np.concatenate(([0], np.cumsum([g.number_of_edges() for g in graphs]))).astype(np.int64)
        cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs), dtype=dt) if xs else np.zeros(0, dt)
        self.node_ent = cat([g.node_id for g in graphs], np.int32)
        self.src = cat([g.src for g in graphs], np.int32)
        self.dst = cat([g.dst for g in graphs], np.int32)
        self.type_s = cat([g.type_s for g in graphs], np.int32)
        self.type_o = cat([g.type_o for g in graphs], np.int32)
        self.graphs = graphs
        self.num_types = int(max(self.type_s.max(), self.type_o.max())) + 1 if len(self.type_s) else 1
        self._dev = {}
        self._node_key = None
        self._row_table = None

    def device_arrays(self, device):
        """The store's edge arrays resident in HBM (uploaded once per device): what renet_induce_edges filters."""
        key = str(torch.device(device))
        d = self._dev.get(key)
        if d is None:
            up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)      # noqa: E731
            d = self._dev[key] = dict(edge_off=up(self.edge_off), src=up(self.src), dst=up(self.dst), type_s=up(self.type_s),
                                      type_o=up(self.type_o))
        return d

    def hot_relations(self, device, n=128):
        """{reverse: device int32 [<= n]}: the relation ids of the type_s (reverse False) / type_o (True) column ranked by
        their frequency over the whole graph_dict.  Relation frequencies are a property of the dataset, so this is
        computed once; the batch-scale gather keeps the first few dozen of these relations' rows in shared memory."""
        key = ('hot', str(torch.device(device)), int(n))
        d = self._dev.get(key)
        if d is None:
            d = {}
            for rev, col in ((False, self.type_s), (True, self.type_o)):
                freq = np.bincount(col.astype(np.int64), minlength=self.num_types)
                order = np.argsort(-freq, kind='stable')
                order = order[freq[order] > 0][:n].astype(np.int32)
                d[rev] = torch.from_numpy(np.ascontiguousarray(order)).to(device)
            self._dev[key] = d
        return d

    def __getitem__(self, t):
        return self.graph_dict[t]

    def __contains__(self, t):
        return t in self.graph_dict

    def keys(self):
        return self.graph_dict.keys()

    def local_rows_many(self, gi, entities):
        """Local rows of (graph index, entity) pairs, vectorised: the store's nodes are sorted by (graph, entity), so
        one searchsorted over a combined key finds them all."""
        gi = np.asarray(gi, dtype=np.int64)
        entities = np.asarray(entities, dtype=np.int64)
        if len(gi) == 0:
            return np.zeros(0, np.int32)
        if self._node_key is None:
            self._key_mul = int(self.node_ent.max()) + 1 if len(self.node_ent) else 1
            owner = np.repeat(np.arange(len(self.times), dtype=np.int64), np.diff(self.node_off))
            self._node_key = owner * self._key_mul + self.node_ent.astype(np.int64)
            if len(self.times) * self._key_mul <= (1 << 26):       # dense (graph, entity) -> row table: 22 MB for ICEWS18
                self._row_table = np.full(len(self.times) * self._key_mul, -1, dtype=np.int32)
                self._row_table[self._node_key] = (np.arange(len(self.node_ent)) - self.node_off[owner]).astype(np.int32)
        if entities.max() >= self._key_mul or entities.min() < 0:
            raise KeyError('entity not present in the graph of its timestamp')
        q = gi * self._key_mul + entities
        if self._row_table is not None:
            rows = self._row_table[q]
            missing = rows < 0
        else:
            pos = np.searchsorted(self._node_key, q)
            missing = (pos >= len(self._node_key)) | (self._node_key[np.minimum(pos, len(self._node_key) - 1)] != q)
            rows = (pos - self.node_off[gi]).astype(np.int32)
        if np.any(missing):
            bad = int(np.flatnonzero(missing)[0])
            raise KeyError('entity %d not present in the graph of timestamp %d' % (int(entities[bad]), int(self.times[gi[bad]])))
        return rows

    def local_rows(self, gi, entities):
        lo = self.node_off[gi]
        ent = self.node_ent[lo:self.node_off[gi + 1]]
        rows = np.searchsorted(ent, entities)
        if np.any(rows >= len(ent)) or np.any(ent[np.minimum(rows, len(ent) - 1)] != entities):
            raise KeyError('entity not present in the graph of timestamp %d' % int(self.times[gi]))
        return rows.astype(np.int32)


class HistoryStore:
    """Histories of a whole split (the reference's pickled train_history_{sub,ob}.txt), flattened, with every
    entity already resolved to its local row in that timestamp's graph."""

    def __init__(self, hist, hist_t, subjects, graph_store, dedupe=True, reverse=None):
        """``reverse`` (optional hint): the edge-type column these histories are used with -- False for subject histories
        (type_s), True for object histories (type_o), model.py:65-78.  With it the batcher also builds layer 2's read-out
        sub-graph ahead of time, on the loader stream.
        hist / hist_t: the reference's per-sample lists (list[n] of list[<=L] of int arrays [k,2] / timestamps);
        subjects: int [n].  Vectorised: one pass over the entries to collect them, everything else in numpy.
        ``dedupe``: the reference's history lists share one array object per (entity, timestamp) among all the samples
        of that entity, so entries are keyed on (array identity, subject) and stored once; pass False for throw-away
        stores of a single batch (``view_from_lists``), where the sort that finds duplicates costs more than it saves."""
        self.gs = gs = graph_store
        self.reverse = reverse
        n = len(hist)
        self.subjects = np.asarray(subjects, dtype=np.int64)
        lens = np.fromiter((len(h) for h in hist), dtype=np.int64, count=n)
        self.samp_off = np.concatenate(([0], np.cumsum(lens))).astype(np.int64)
        total = int(self.samp_off[-1])
        arrays = [a for h in hist for a in h]
        flat_t = np.fromiter((int(t) for ht in hist_t for t in ht), dtype=np.int64, count=total)
        flat_s = np.repeat(self.subjects, lens)
        if dedupe and total:
            ids = np.fromiter(map(id, arrays), dtype=np.int64, count=total)
            order = np.lexsort((flat_s, ids))
            new = np.ones(total, dtype=bool)
            new[1:] = (ids[order][1:] != ids[order][:-1]) | (flat_s[order][1:] != flat_s[order][:-1])
            first = order[new]                                  # one representative row per distinct entry
            entry_of_sorted = np.cumsum(new) - 1
            samp_entry = np.empty(total, dtype=np.int64)
            samp_entry[order] = entry_of_sorted
        else:
            first = np.arange(total, dtype=np.int64)
            samp_entry = first.copy()
        self.samp_entry = samp_entry
        ent_t, ent_s = flat_t[first], flat_s[first]
        gi = np.searchsorted(gs.times, ent_t)
        if total and (np.any(gi >= len(gs.times)) or np.any(gs.times[np.minimum(gi, len(gs.times) - 1)] != ent_t)):
            raise KeyError('history refers to a timestamp that is not in the graph store')
        self.ent_graph = gi.astype(np.int32)
        self.ent_srow = gs.local_rows_many(gi, ent_s)
        ent_arrays = arrays if len(first) == total and not dedupe else [arrays[i] for i in first]
        ent_len = np.fromiter(map(len, ent_arrays), dtype=np.int64, count=len(ent_arrays))
        self.ent_off = np.concatenate(([0], np.cumsum(ent_len))).astype(np.int64)
        if len(ent_arrays):
            nbr_ent = np.concatenate(ent_arrays).reshape(-1, 2)[:, 1].astype(np.int64)      # one concatenate, then column 1
            self.nbr_row = gs.local_rows_many(np.repeat(gi, ent_len), nbr_ent)
        else:
            self.nbr_row = np.zeros(0, np.int32)
        self._keepalive = hist        # array identities are the entry keys: keep the arrays alive

    def select(self, sample_idx, groups=None):
        return HistoryView(self, np.ascontiguousarray(sample_idx, dtype=np.int64), groups)


class HistoryView:
    """A batch = indices into a HistoryStore.  Passed where the reference passes (s_hist, s_hist_t).

    ``groups`` (optional, one int per selected sample): isolation groups.  The batched history graph then has one component
    per distinct (group, timestamp) instead of one per timestamp, so the samples of a group are encoded exactly as if they
    were batched alone (renet_host_plan_batch_grouped); the reference's predict encodes every (entity, relation) history
    alone.  Only the device batcher takes groups."""

    def __init__(self, store, sample_idx, groups=None):
        self.store, self.sample_idx = store, sample_idx
        self.groups = None
        if groups is not None:
            self.groups = np.ascontiguousarray(groups, dtype=np.int64).reshape(-1)
            if len(self.groups) != len(sample_idx):
                raise ValueError('HistoryView: %d samples but %d groups' % (len(sample_idx), len(self.groups)))

    def __len__(self):
        return len(self.sample_idx)

    def total_length(self):
        so = self.store.samp_off
        return int((so[self.sample_idx + 1] - so[self.sample_idx]).sum())


def view_from_lists(hist, hist_t, subjects, graph_store):
    """The reference's per-batch inputs (s_hist, s_hist_t, s) -> a HistoryView over a throw-away store, so that a batch
    given as Python lists goes through the C++ / device batcher instead of the numpy path (5-8 ms instead of 50-100 ms
    per direction at batch 1024)."""
    subjects = np.asarray(subjects).reshape(-1)
    return HistoryStore(hist, hist_t, subjects, graph_store, dedupe=False).select(np.arange(len(hist)))


class _Staging:
    """Ring of pinned int32 staging buffers; a buffer is reused only after the H2D copy issued from it has
    completed (event)."""

    def __init__(self, n=3, words=1 << 21):
        self.bufs = [torch.empty(words, dtype=torch.int32).pin_memory() for _ in range(n)]
        self.events = [None] * n
        self.i = 0

    def next(self, min_words=0):
        self.i = (self.i + 1) % len(self.bufs)
        ev = self.events[self.i]
        if ev is not None:
            ev.synchronize()
        if self.bufs[self.i].numel() < min_words:
            self.bufs[self.i] = torch.empty(int(min_words * 1.5), dtype=torch.int32).pin_memory()
        return self.i, self.bufs[self.i]


_staging = {}
_PINNED_POOL = __import__('collections').deque()


def reserve_pinned(n, words=1 << 21):
    """Make sure the process-wide pool holds at least ``n`` pinned staging buffers.  Pinning is expensive (cudaHostAlloc
    of 8 MB: 4-10 ms, and it can stall the device), so a loader should never have to do it in the middle of a run."""
    while len(_PINNED_POOL) < n:
        _PINNED_POOL.append(torch.empty(words, dtype=torch.int32).pin_memory())


def assemble_view_raw(view, out, sort=True):
    """Run the C++ batcher into the int32 numpy buffer ``out`` (host only, no CUDA).  Returns None when
    the buffer is too small (sizes[6] words are needed), else a dict of sizes + small host arrays."""
    if view.groups is not None:
        raise ValueError('isolation groups need the device batcher (device_edges=True)')
    L = _lib.lib()
    hs, gs = view.store, view.store.gs
    B = len(view.sample_idx)
    s_idx = np.empty(B, dtype=np.int64)
    comp_graph = np.empty(len(gs.times), dtype=np.int32)
    bsz = np.zeros(MAX_LEN, dtype=np.int32)
    sizes = np.zeros(10, dtype=np.int64)
    rc = L.renet_host_assemble_batch(
        len(gs.times), _p(gs.node_off), _p(gs.node_ent), _p(gs.edge_off), _p(gs.src), _p(gs.dst), _p(gs.type_s),
        _p(gs.type_o), _p(hs.samp_off), _p(hs.samp_entry), _p(hs.ent_graph), _p(hs.ent_srow), _p(hs.ent_off), _p(hs.nbr_row),
        _p(view.sample_idx), B, int(sort), gs.num_types, N_HOT, _p(s_idx), _p(out), out.size, _p(comp_graph), _p(bsz), MAX_LEN, _p(sizes))
    if rc == 1:
        return {'need_words': int(sizes[6])}
    _lib.check(rc, 'renet_host_assemble_batch')
    N, E, S, Q, G, max_len, words = (int(x) for x in sizes[:7])
    return dict(N=N, E=E, S=S, Q=Q, G=G, max_len=max_len, words=words, s_idx=s_idx, comp_graph=comp_graph[:G],
                batch_sizes=bsz[:max_len].copy(), R2=gs.num_types, n_hot_s=int(sizes[7]), n_hot_o=int(sizes[8]), B=B)


def split_raw(buf, r):
    """Views into the staged buffer (numpy or torch), in the layout renet_host_assemble_batch documents."""
    N, E, S, Q = r['N'], r['E'], r['S'], r['Q']
    o = 0
    out = {}
    for name, n in (('node_ent', N), ('row_ptr', N + 1), ('col_src', E), ('col_type_s', E), ('col_type_o', E),
                    ('norm', N), ('readout', S), ('row_comp', S), ('row_seq', S), ('seq_start', Q), ('seq_len', Q),
                    ('packed_row', S), ('comp_ptr', r['G'] + 1), ('comp_order', r['G']), ('rel_slot_s', r['R2']),
                    ('hot_s', N_HOT), ('rel_slot_o', r['R2']), ('hot_o', N_HOT), ('s_idx', r['B']),
                    ('comp_graph', r['G'])):
        out[name] = buf[o:o + n]
        o += n
    return out


def plan_view_raw(view, out, sort=True):
    """Host half of the device batcher (renet_host_plan_batch_grouped, with the view's isolation groups if it has any)
    into the int32 numpy buffer ``out``."""
    L = _lib.lib()
    hs, gs = view.store, view.store.gs
    B = len(view.sample_idx)
    s_idx = np.empty(B, dtype=np.int64)
    bsz = np.zeros(MAX_LEN, dtype=np.int32)
    sizes = np.zeros(10, dtype=np.int64)
    groups = _p(view.groups) if view.groups is not None else None
    rc = L.renet_host_plan_batch_grouped(
        len(gs.times), _p(gs.node_off), _p(gs.node_ent), _p(gs.edge_off), _p(hs.samp_off), _p(hs.samp_entry), _p(hs.ent_graph),
        _p(hs.ent_srow), _p(hs.ent_off), _p(hs.nbr_row), _p(view.sample_idx), groups, B, int(sort), _p(s_idx), _p(out),
        out.size, _p(bsz), MAX_LEN, _p(sizes))
    if rc == 1:
        return {'need_words': int(sizes[6])}
    _lib.check(rc, 'renet_host_plan_batch')
    N, E_cand, S, Q, G, max_len, words, M = (int(x) for x in sizes[:8])
    return dict(N=N, E_cand=E_cand, S=S, Q=Q, G=G, max_len=max_len, words=words, M=M, s_idx=s_idx,
                batch_sizes=bsz[:max_len].copy(), B=B, plan=True)


def split_plan(buf, r):
    """Views into a staged plan buffer, in the layout renet_host_plan_batch documents."""
    o = 0
    out = {}
    for name, n in (('newid', r['M']), ('node_ent', r['N']), ('readout', r['S']), ('row_comp', r['S']), ('row_seq', r['S']),
                    ('seq_start', r['Q']), ('seq_len', r['Q']), ('packed_row', r['S']), ('s_idx', r['B']),
                    ('comp_graph', r['G']), ('mark_off', r['G'] + 1), ('cand_off', r['G'] + 1)):
        out[name] = buf[o:o + n]
        o += n
    return out


class NativeLoader:
    """C++ worker threads (renet_loader_*) running batch jobs ahead of the consumer, without the GIL."""

    def __init__(self, workers):
        self.L = _lib.lib()
        self.h = self.L.renet_loader_create(int(workers))
        if not self.h:
            raise RuntimeError('renet_loader_create failed')

    def close(self):
        if self.h:
            self.L.renet_loader_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def submit(self, view, out, sort, device_edges):
        """Enqueue the host work of one batch into the int32 numpy buffer ``out``; returns the job record that finish()
        takes (it keeps every array the C++ job writes alive)."""
        if view.groups is not None:
            raise ValueError('NativeLoader: isolation groups are not supported; use assemble_view')
        hs, gs = view.store, view.store.gs
        B = len(view.sample_idx)
        job = dict(view=view, out=out, sort=sort, device_edges=device_edges, B=B, s_idx=np.empty(B, dtype=np.int64),
                   bsz=np.zeros(MAX_LEN, dtype=np.int32), sizes=np.zeros(10, dtype=np.int64),
                   comp_graph=np.empty(len(gs.times), dtype=np.int32))
        if device_edges:
            t = self.L.renet_loader_submit_plan(
                self.h, len(gs.times), _p(gs.node_off), _p(gs.node_ent), _p(gs.edge_off), _p(hs.samp_off), _p(hs.samp_entry),
                _p(hs.ent_graph), _p(hs.ent_srow), _p(hs.ent_off), _p(hs.nbr_row), _p(view.sample_idx), B, int(sort),
                _p(job['s_idx']), _p(out), out.size, _p(job['bsz']), MAX_LEN, _p(job['sizes']))
        else:
            t = self.L.renet_loader_submit_assemble(
                self.h, len(gs.times), _p(gs.node_off), _p(gs.node_ent), _p(gs.edge_off), _p(gs.src), _p(gs.dst), _p(gs.type_s),
                _p(gs.type_o), _p(hs.samp_off), _p(hs.samp_entry), _p(hs.ent_graph), _p(hs.ent_srow), _p(hs.ent_off),
                _p(hs.nbr_row), _p(view.sample_idx), B, int(sort), gs.num_types, N_HOT, _p(job['s_idx']), _p(out), out.size,
                _p(job['comp_graph']), _p(job['bsz']), MAX_LEN, _p(job['sizes']))
        if t < 0:
            raise RuntimeError('renet_loader_submit failed')
        job['ticket'] = t
        return job

    def finish(self, job):
        """Wait for the job; returns the dict plan_view_raw / assemble_view_raw return."""
        rc = self.L.renet_loader_wait(self.h, job['ticket'])
        sizes = job['sizes']
        if rc == 1:
            return {'need_words': int(sizes[6])}
        _lib.check(rc, 'renet_loader job')
        if job['device_edges']:
            N, E_cand, S, Q, G, max_len, words, M = (int(x) for x in sizes[:8])
            return dict(N=N, E_cand=E_cand, S=S, Q=Q, G=G, max_len=max_len, words=words, M=M, s_idx=job['s_idx'],
                        batch_sizes=job['bsz'][:max_len].copy(), B=job['B'], plan=True)
        N, E, S, Q, G, max_len, words = (int(x) for x in sizes[:7])
        gs = job['view'].store.gs
        return dict(N=N, E=E, S=S, Q=Q, G=G, max_len=max_len, words=words, s_idx=job['s_idx'],
                    comp_graph=job['comp_graph'][:G], batch_sizes=job['bsz'][:max_len].copy(), R2=gs.num_types,
                    n_hot_s=int(sizes[7]), n_hot_o=int(sizes[8]), B=job['B'])


_E_PINNED = __import__('collections').deque()       # pool of pinned int32[1] read-back slots
_LOADER_STREAMS = {}


def _loader_stream(device):
    key = str(torch.device(device))
    st = _LOADER_STREAMS.get(key)
    if st is None:
        st = _LOADER_STREAMS[key] = torch.cuda.Stream(device=device)
    return st


def _upload_plan(view, buf, r, device):
    """Device part of the device batcher (caller's thread / current stream): one pinned H2D copy of the plan, then
    renet_induce_edges builds the CSR on the GPU from the resident graph store; the edge count comes back
    asynchronously (graph.E resolves it on demand)."""
    hb = HistoryBatch()
    hb.s_idx, hb.num_seq, hb.S = r['s_idx'], r['Q'], r['S']
    if r['S'] == 0:
        hb.graph, hb.seq_len = None, np.zeros(0, np.int64)
        return hb, None
    L = _lib.lib()
    gs = view.store.gs
    ga = gs.device_arrays(device)
    words, N, E_cand = r['words'], r['N'], r['E_cand']
    # the copy and the CSR build run on a loader stream, so they overlap the previous step's kernels on the caller's
    # stream; the caller's stream waits on `ready` before it touches the batch
    main = torch.cuda.current_stream(device)
    ls = _loader_stream(device)
    with torch.cuda.stream(ls):
        dev = buf[:words].to(device, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(ls)
        d = split_plan(dev, r)
        h = split_plan(buf.numpy(), r)
        ws_bytes = int(L.renet_induce_workspace_bytes(E_cand))
        # one allocation: row_ptr[N+1] col_src col_type_s col_type_o [E_cand each] norm[N] e_count[1] + workspace
        blob = torch.empty(N + 1 + 3 * E_cand + N + 1 + ws_bytes // 4 + 64, dtype=torch.int32, device=device)
        o = 0
        parts = {}
        for name, n in (('row_ptr', N + 1), ('col_src', E_cand), ('col_type_s', E_cand), ('col_type_o', E_cand), ('norm', N),
                        ('e_count', 1)):
            parts[name] = blob[o:o + n]
            o += n
        o = (o + 63) // 64 * 64                      # 256-byte aligned workspace
        ws = blob[o:]
        P = _lib.ptr
        rc = L.renet_induce_edges(P(ga['edge_off']), P(ga['src']), P(ga['dst']), P(ga['type_s']), P(ga['type_o']),
                                  P(d['comp_graph']), P(d['mark_off']), P(d['cand_off']), P(d['newid']), r['G'], N, E_cand,
                                  P(parts['row_ptr']), P(parts['col_src']), P(parts['col_type_s']), P(parts['col_type_o']),
                                  P(parts['norm']), P(parts['e_count']), P(ws), ws.numel() * 4, _lib.stream())
        _lib.check(rc, 'renet_induce_edges')
    g = BatchedHistoryGraph.__new__(BatchedHistoryGraph)
    g.device, g.N = torch.device(device), N
    g.E_cap = E_cand
    g.node_ent, g.row_ptr = d['node_ent'], parts['row_ptr']
    g.col_src, g.col_type_s, g.col_type_o = parts['col_src'], parts['col_type_s'], parts['col_type_o']
    g.norm = parts['norm'].view(torch.float32)
    g.comp_sizes = None
    g.h2d_bytes = words * 4
    g.ndata = _Frame(norm=g.norm.view(-1, 1), id=g.node_ent.view(-1, 1))
    g.h_index = g.h_table = None
    g._bwd = {}
    g.G, g.comp = r['G'], None
    g.seq_len_dev = d['seq_len']
    g.hot = gs.hot_relations(device)
    g._keep = (blob, dev)
    with torch.cuda.stream(ls):
        rev = getattr(view.store, 'reverse', None)
        sub = None
        if rev is not None:
            # the store knows which edge-type column its histories are used with (subject histories: type_s, object
            # histories: type_o, model.py:65-78): layer 2's read-out sub-graph is built here, on the loader stream too
            sub = g.readout_sub(d['readout'], rev)
        ready = torch.cuda.Event()
        ready.record(ls)
        if not _E_PINNED:
            _lib.pinned_slots(_E_PINNED, 1)
        e_host = _E_PINNED.pop()
        e_host.copy_(parts['e_count'], non_blocking=True)
        e_ev = torch.cuda.Event()
        e_ev.record(ls)
    main.wait_event(ready)
    dev.record_stream(main)          # allocated on the loader stream, consumed on the caller's
    blob.record_stream(main)
    if sub is not None:
        for t in sub._keep:
            t.record_stream(main)
    g._E_pending = PendingCount(e_ev, e_host, _E_PINNED.append)
    hb.graph = g
    hb.readout, hb.row_glob, hb.row_seq = d['readout'], d['row_comp'], d['row_seq']
    hb.seq_start, hb.packed_row = d['seq_start'], d['packed_row']
    hb.readout_host = h['readout'].astype(np.int64)
    hb.seq_len = h['seq_len'].astype(np.int64)
    hb.batch_sizes = r['batch_sizes']
    hb.times = gs.times[h['comp_graph']]
    hb.h2d_bytes = words * 4
    hb.s_idx_dev, hb.comp_graph_dev = d['s_idx'], d['comp_graph']
    hb.graph_store = gs
    return hb, ev


def _stage(view, buf_holder, sort, device_edges=False):
    """Host part: run the C++ batcher (or, with device_edges, only its planning half) into a pinned buffer (grows it
    when needed).  Thread-safe per buffer."""
    fn = plan_view_raw if device_edges else assemble_view_raw
    r = fn(view, buf_holder[0].numpy(), sort)
    if 'need_words' in r:
        buf_holder[0] = torch.empty(int(r['need_words'] * 1.5), dtype=torch.int32).pin_memory()
        r = fn(view, buf_holder[0].numpy(), sort)
    return r


def _upload(view, buf, r, device):
    """Device part (caller's thread / current stream): one pinned H2D copy, then slice it into the batch."""
    if r.get('plan'):
        return _upload_plan(view, buf, r, device)
    hb = HistoryBatch()
    hb.s_idx, hb.num_seq, hb.S = r['s_idx'], r['Q'], r['S']
    if r['S'] == 0:
        hb.graph, hb.seq_len = None, np.zeros(0, np.int64)
        return hb, None
    words = r['words']
    dev = buf[:words].to(device, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    d = split_raw(dev, r)
    h = split_raw(buf.numpy(), r)
    g = BatchedHistoryGraph.__new__(BatchedHistoryGraph)
    g.device, g.N, g.E = torch.device(device), r['N'], r['E']
    g.node_ent, g.row_ptr = d['node_ent'], d['row_ptr']
    g.col_src, g.col_type_s, g.col_type_o = d['col_src'], d['col_type_s'], d['col_type_o']
    g.norm = d['norm'].view(torch.float32)
    g.comp_sizes = None
    g.h2d_bytes = words * 4
    g.ndata = _Frame(norm=g.norm.view(-1, 1), id=g.node_ent.view(-1, 1))
    g.h_index = g.h_table = None
    g._bwd = {}
    g.G = r['G']
    g.comp = {False: (d['comp_ptr'], d['comp_order'], d['rel_slot_s'], d['hot_s'], r['n_hot_s']),
              True: (d['comp_ptr'], d['comp_order'], d['rel_slot_o'], d['hot_o'], r['n_hot_o'])}
    g.seq_len_dev = d['seq_len']
    g.hot = view.store.gs.hot_relations(device)
    hb.graph = g
    hb.readout, hb.row_glob, hb.row_seq = d['readout'], d['row_comp'], d['row_seq']
    hb.seq_start, hb.packed_row = d['seq_start'], d['packed_row']
    hb.readout_host = h['readout'].astype(np.int64)
    hb.seq_len = h['seq_len'].astype(np.int64)
    hb.batch_sizes = r['batch_sizes']
    hb.times = view.store.gs.times[r['comp_graph']]
    hb.h2d_bytes = words * 4
    hb.s_idx_dev, hb.comp_graph_dev = d['s_idx'], d['comp_graph']     # device copies: no pageable H2D later
    hb.graph_store = view.store.gs
    return hb, ev


DEVICE_EDGES = True      # build the batched CSR on the GPU (renet_induce_edges); False = all-host C++ batcher


def assemble_view(view, device, sort=True, device_edges=None):
    """HistoryView -> HistoryBatch on ``device``: host plan + one pinned H2D copy + renet_induce_edges on the GPU
    (default), or the all-host C++ batcher + one pinned H2D copy (device_edges=False; not for views with groups)."""
    if device_edges is None:
        device_edges = DEVICE_EDGES
    if view.groups is not None and not device_edges:
        raise ValueError('isolation groups need the device batcher (device_edges=True)')
    st = _staging.get(str(device))
    if st is None:
        st = _staging[str(device)] = _Staging()
    slot, buf = st.next()
    holder = [buf]
    r = _stage(view, holder, sort, device_edges)
    st.bufs[slot] = holder[0]
    hb, ev = _upload(view, holder[0], r, device)
    st.events[slot] = ev
    return hb


def prefetch(view_groups, device, depth=2, workers=4, sort=True, inner_threads=1, device_edges=None):
    """Pipeline the host batching: ``view_groups`` is an iterable of tuples of HistoryViews (one tuple per step,
    e.g. (subject view, object view)); yields tuples of HistoryBatches on ``device``.  While the consumer runs
    step i on the GPU, native worker threads (renet_loader_*, no GIL) prepare steps i+1 .. i+depth into their own
    pinned staging buffers; the H2D copy (and, with the device batcher, the CSR build) is issued from the consumer's
    thread when the batch is handed over."""
    import collections
    if device_edges is None:
        device_edges = DEVICE_EDGES
    prev_threads = None
    if inner_threads is not None:          # many concurrent batcher calls: fewer threads inside each
        prev_threads = _lib.lib().renet_set_host_threads(int(inner_threads))
    free = _PINNED_POOL          # pinned staging buffers are expensive to create (~4 ms each): pooled per process
    reserve_pinned(2 * (depth + 3) + 2)      # two views per step in flight for depth steps + uploads not yet retired
    loader = NativeLoader(workers)
    pending = collections.deque()
    it = iter(view_groups)

    def start(view):
        try:
            buf = free.pop()
        except IndexError:
            buf = torch.empty(1 << 21, dtype=torch.int32).pin_memory()
        return [buf], loader.submit(view, buf.numpy(), sort, device_edges)

    def submit():
        try:
            grp = next(it)
        except StopIteration:
            return False
        pending.append([start(v) for v in grp])
        return True

    try:
        for _ in range(depth):
            if not submit():
                break
        in_flight = collections.deque()       # (event, buffer) of uploads whose pinned buffer is not reusable yet
        while pending:
            jobs = pending.popleft()
            out = []
            for holder, job in jobs:
                r = loader.finish(job)
                if 'need_words' in r:            # staging buffer too small: grow it and redo this batch synchronously
                    holder[0] = torch.empty(int(r['need_words'] * 1.5), dtype=torch.int32).pin_memory()
                    r = _stage(job['view'], holder, sort, device_edges)
                hb, ev = _upload(job['view'], holder[0], r, device)
                out.append(hb)
                in_flight.append((ev, holder[0]))
            submit()
            while in_flight and (in_flight[0][0] is None or in_flight[0][0].query()):
                free.append(in_flight.popleft()[1])
            yield tuple(out)
        for ev, buf in in_flight:          # hand the remaining buffers back once their copies have completed
            if ev is not None:
                ev.synchronize()
            free.append(buf)
    finally:
        for jobs in pending:               # consumer stopped early: the jobs still own their buffers until they ran
            for holder, job in jobs:
                loader.finish(job)
        loader.close()
        if prev_threads is not None:
            _lib.lib().renet_set_host_threads(prev_threads)
