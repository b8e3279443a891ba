"""DGL-free graph containers for the RE-Net hot path.

The reference stores one ``dgl.DGLGraph`` per timestamp in ``graph_dict`` (built by
utils.get_big_graph, reference utils.py:68-87) and batches vertex-induced sub-graphs of them per
training batch (utils.py:115-131, 158-181, 238).  DGL 0.4 is neither installable nor needed here:

* ``HistoryGraph``  -- one timestamp's graph.  Exposes the attributes the reference code touches
  (``ids``, ``ndata['id'|'norm']``, ``edata['type_s'|'type_o']``, ``number_of_nodes()``, ``edges()``,
  ``in_degrees()``) and keeps int32 numpy arrays, edges pre-sorted by destination, so that batching is
  pure array slicing and the batched graph is born in CSR form.
* ``BatchedHistoryGraph`` -- the disjoint union handed to the RGCN layers: device-resident CSR by
  destination (+ lazily the CSR by source and the relation-grouped edge list the backward kernels
  need).  ``ndata`` is dict-like (``['h']``, ``pop('h')``) as the reference's aggregator expects
  (Aggregator.py:139).

``as_history_graph`` adapts any object with the DGL 0.4 surface (real DGL, or the test shim).
"""
import numpy as np
import torch

from . import _lib


class _Frame(dict):
    pass


class HistoryGraph:
    """Graph of one timestamp: what reference utils.get_big_graph returns (utils.py:68-87)."""

    def __init__(self, node_id, src, dst, type_s, type_o):
        self.node_id = np.ascontiguousarray(node_id, dtype=np.int64)     # entity id per local row
        n = len(self.node_id)
        src = np.asarray(src, dtype=np.int32)
        dst = np.asarray(dst, dtype=np.int32)
        # COO in insertion order (DGL-compatible view) ...
        self._coo = (src, dst, np.asarray(type_s, dtype=np.int32), np.asarray(type_o, dtype=np.int32))
        # ... and a destination-sorted copy (stable) used by the batching code
        order = np.argsort(dst, kind='stable')
        self.src = np.ascontiguousarray(src[order])
        self.dst = np.ascontiguousarray(dst[order])
        self.type_s = np.ascontiguousarray(self._coo[2][order])
        self.type_o = np.ascontiguousarray(self._coo[3][order])
        self.ids = {int(e): i for i, e in enumerate(self.node_id)}       # utils.py:82-86
        deg = np.bincount(self.dst, minlength=n).astype(np.float32)
        deg[deg == 0] = 1.0
        self.norm = (np.float32(1.0) / deg).astype(np.float32)           # utils.py:89-93
        self._sorted = bool(np.all(self.node_id[1:] > self.node_id[:-1])) if n > 1 else True
        self.start_id = 0

    # ---- the DGL-ish surface the reference's code reads ------------------------------------------
    @property
    def ndata(self):
        return _Frame(id=torch.from_numpy(self.node_id).view(-1, 1),
                      norm=torch.from_numpy(self.norm).view(-1, 1))

    @property
    def edata(self):
        return _Frame(type_s=torch.from_numpy(self._coo[2].astype(np.int64)),
                      type_o=torch.from_numpy(self._coo[3].astype(np.int64)))

    def number_of_nodes(self):
        return len(self.node_id)

    def number_of_edges(self):
        return len(self.src)

    def edges(self):
        return (torch.from_numpy(self._coo[0].astype(np.int64)), torch.from_numpy(self._coo[1].astype(np.int64)))

    def in_degrees(self, nodes=None):
        deg = torch.from_numpy(np.bincount(self.dst, minlength=len(self.node_id)))
        return deg if nodes is None else deg[torch.as_tensor(list(nodes), dtype=torch.long)]

    def to(self, device):
        return self

    # ---- batching helpers ---------------------------------------------------------------------
    def rows_of(self, entities):
        """local rows of an int64 array of entity ids (all must be present)."""
        if self._sorted:
            return np.searchsorted(self.node_id, entities)
        return np.asarray([self.ids[int(e)] for e in entities], dtype=np.int64)


def get_big_graph(data, num_rels):
    """Same contract as reference utils.get_big_graph (utils.py:68-87): triples (s, r, o) of ONE
    timestamp -> graph with both edge directions; type_s = [r.., r+R..], type_o = [r+R.., r..]."""
    data = np.asarray(data, dtype=np.int64)
    s, r, o = data[:, 0], data[:, 1], data[:, 2]
    uniq_v, inv = np.unique(np.stack((s, o)), return_inverse=True)
    ls, lo = np.reshape(inv, (2, -1))
    return HistoryGraph(uniq_v, np.concatenate((ls, lo)), np.concatenate((lo, ls)),
                        np.concatenate((r, r + num_rels)), np.concatenate((r + num_rels, r)))


def as_history_graph(g):
    """Adapt a DGL-0.4-style graph object (real DGL or a stand-in) to HistoryGraph; cached on g."""
    if isinstance(g, HistoryGraph):
        return g
    cached = getattr(g, '_renet_b200_graph', None)
    if cached is not None:
        return cached
    src, dst = g.edges()
    hg = HistoryGraph(g.ndata['id'].view(-1).cpu().numpy(), src.cpu().numpy(), dst.cpu().numpy(),
                      g.edata['type_s'].cpu().numpy(), g.edata['type_o'].cpu().numpy())
    try:
        g._renet_b200_graph = hg
    except Exception:
        pass
    return hg


class PendingCount:
    """An integer the GPU produces: (event, pinned int32[1]) of an asynchronous device->host read-back; value() waits
    for the event once, caches the number and hands the pinned slot back to its pool."""

    def __init__(self, event, pinned, release=None):
        self._ev, self._pinned, self._release, self._v = event, pinned, release, None

    def value(self):
        if self._v is None:
            self._ev.synchronize()
            self._v = int(self._pinned[0])
            if self._release is not None:
                self._release(self._pinned)
            self._ev = self._pinned = self._release = None
        return self._v


class _KnownCount:
    def __init__(self, v):
        self._v = int(v)

    def value(self):
        return self._v


class BatchedHistoryGraph:
    """Disjoint union of induced sub-graphs, device-resident, CSR by destination.

    Equivalent of ``dgl.batch(g_list)`` + ``move_dgl_to_cuda`` (reference utils.py:237-241)."""

    def __init__(self, node_ent, norm, row_ptr, col_src, col_type_s, col_type_o, device):
        self.device = torch.device(device)
        self.N = int(len(node_ent))
        self.E = int(len(col_src))
        # one pinned staging buffer -> one H2D copy
        parts = [node_ent, row_ptr, col_src, col_type_s, col_type_o]
        i32 = np.concatenate([np.asarray(p).astype(np.int32) for p in parts])
        dev = _to_device(torch.from_numpy(i32), self.device)
        o = 0
        self.node_ent = dev[o:o + self.N]; o += self.N
        self.row_ptr = dev[o:o + self.N + 1]; o += self.N + 1
        self.col_src = dev[o:o + self.E]; o += self.E
        self.col_type_s = dev[o:o + self.E]; o += self.E
        self.col_type_o = dev[o:o + self.E]
        self.norm = _to_device(torch.from_numpy(np.ascontiguousarray(norm, dtype=np.float32)), self.device)
        self.h2d_bytes = i32.nbytes + self.N * 4
        self.ndata = _Frame(norm=self.norm.view(-1, 1), id=self.node_ent.view(-1, 1))
        self.h_index = None          # when set, ndata['h'] is virtual: H = table[h_index]
        self.h_table = None
        self._bwd = {}

    # ---- edge count: known on the host for host-assembled batches; for device-assembled ones (hoststore, device
    # batcher) it is produced on the GPU and read back lazily, so nothing on the forward path waits for it ------------
    _E = None
    _E_pending = None       # PendingCount of the asynchronous read-back (device-assembled batches)
    E_cap = None            # capacity of the col_* arrays (>= E); launch argument while E is still in flight
    has_edge = False        # E >= 1 is known on the host without waiting for E (hoststore._first_entry_has_edge)

    @property
    def E(self):
        if self._E is None:
            self._E = self._E_pending.value()
            self._E_pending = None
            self.col_src, self.col_type_s, self.col_type_o = (x[:self._E] for x in (self.col_src, self.col_type_s, self.col_type_o))
        return self._E

    def edge_count_handle(self):
        """Something with ``.value()`` that yields E later WITHOUT keeping the graph (and its device memory) alive."""
        return self._E_pending if self._E is None else _KnownCount(self._E)

    @E.setter
    def E(self, v):
        self._E = int(v)

    @property
    def E_launch(self):
        """E when it is known without waiting, else the capacity bound (the kernels walk row_ptr, not E)."""
        return self._E if self._E is not None else self.E_cap

    def number_of_nodes(self):
        return self.N

    def number_of_edges(self):
        return self.E

    def col_type(self, reverse):
        """edge-type column the reference selects with ``reverse`` (RGCN.py:80-85)."""
        return self.col_type_o if reverse else self.col_type_s

    def hot_rel(self, reverse):
        """The dataset's most frequent relation ids of that type column (device int32, most frequent first) when the graph
        came from a GraphStore, else None: the batch-scale gather keeps those relations' rows in shared memory
        (renet_rgcn_gather_hot); without a list every CTA ranks the relations of its own edges."""
        hot = getattr(self, 'hot', None)
        return None if hot is None else hot[bool(reverse)]

    def coo_dst(self):
        if 'dst' not in self._bwd:
            self.E          # device-assembled batch: resolve the asynchronous edge count first (trims col_* to E entries)
            counts = (self.row_ptr[1:] - self.row_ptr[:-1]).long()
            self._bwd['dst'] = torch.repeat_interleave(
                torch.arange(self.N, device=self.device, dtype=torch.int32), counts)
        return self._bwd['dst']

    def readout_sub(self, readout, reverse):
        """The read-out sub-graph layer 2 runs on (ReadoutSubgraph), built once per type column."""
        key = ('sub', bool(reverse))
        if key not in self._bwd:
            self._bwd[key] = ReadoutSubgraph(self, readout, reverse)
        return self._bwd[key]

    def backward_structs(self, reverse, num_types):
        """(t_row_ptr, t_col_dst, t_col_type, rel_ptr, rel_src, rel_dst) for the backward kernels."""
        key = ('bwd', bool(reverse), int(num_types))
        if key not in self._bwd:
            # the device batcher returns E asynchronously and leaves col_* at capacity E_cand with an uninitialised tail:
            # reading self.E waits for the count and trims the columns, so build_csr never sees the tail
            assert self.E == int(self.col_src.numel())
            dst = self.coo_dst()
            et = self.col_type(reverse)
            t_row_ptr, t_col_dst, t_col_type, _ = build_csr(self.col_src, dst, et, self.N)
            # group by relation: key = etype, payload = (src, dst)
            rel_ptr, rel_src, rel_dst, _ = build_csr(et, self.col_src, dst, num_types)
            self._bwd[key] = (t_row_ptr, t_col_dst, t_col_type, rel_ptr, rel_src, rel_dst)
        return self._bwd[key]


_CNT_PINNED = __import__('collections').deque()       # pool of pinned int32[2] read-back slots


class ReadoutSubgraph:
    """Layer 2's graph: only the edges whose destination is a read-out node (reference Aggregator.py:139-140 keeps
    nothing else of layer 2's output).  Built on the device by renet_readout_subgraph, on the current stream, without
    waiting for anything: capacities are S destinations and the parent's edge capacity; the real sizes (U distinct
    read-out nodes, E2 edges) come back asynchronously and are only needed by backward.

    Destinations are compact (row u <-> node uniq[u]); sources keep the parent's node ids (rows of H1).  Quacks like
    BatchedHistoryGraph for the layer kernels: N (destination rows), N_src, row_ptr, col_src, col_type(), norm, E_launch."""

    def __init__(self, g, readout, reverse):
        L = _lib.lib()
        dev = g.device
        S = int(readout.numel())
        self.device, self.N, self.N_src, self.reverse = dev, S, g.N, bool(reverse)
        self._hot = g.hot_rel(reverse) if hasattr(g, 'hot_rel') else None
        self.E_cap = int(g.col_src.numel())
        i32 = torch.empty(3 * S + (S + 1) + 2 * self.E_cap + 2, dtype=torch.int32, device=dev)
        o = 0
        parts = {}
        for name, n in (('uniq', S), ('readout_c', S), ('row_ptr', S + 1), ('col_src', self.E_cap), ('col_type', self.E_cap),
                        ('norm', S), ('counts', 2)):
            parts[name] = i32[o:o + n]
            o += n
        self.uniq, self.readout_c, self.row_ptr = parts['uniq'], parts['readout_c'], parts['row_ptr']
        self.col_src, self._col_type, self.counts = parts['col_src'], parts['col_type'], parts['counts']
        self.norm = parts['norm'].view(torch.float32)
        nbytes = int(L.renet_readout_subgraph_workspace_bytes(g.N, S))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        P = _lib.ptr
        rc = L.renet_readout_subgraph(P(readout), S, g.N, P(g.row_ptr), P(g.col_src), P(g.col_type(reverse)), P(g.norm),
                                      P(self.uniq), P(self.readout_c), P(self.row_ptr), P(self.col_src), P(self._col_type),
                                      P(self.norm), P(self.counts), P(ws), nbytes, _lib.stream())
        _lib.check(rc, 'renet_readout_subgraph')
        if not _CNT_PINNED:
            _lib.pinned_slots(_CNT_PINNED, 2)
        host = _CNT_PINNED.pop()
        host.copy_(self.counts, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._pending, self._host = ev, host
        self._sizes = None
        self._keep = (i32, ws)
        self._bwd = {}

    def sizes(self):
        """(U, E2): waits for the asynchronous read-back once."""
        if self._sizes is None:
            self._pending.synchronize()
            self._sizes = (int(self._host[0]), int(self._host[1]))
            _CNT_PINNED.append(self._host)
            self._pending = self._host = None
        return self._sizes

    @property
    def E(self):
        return self.sizes()[1]

    @property
    def E_launch(self):
        return self.E_cap

    def hot_rel(self, reverse):
        assert bool(reverse) == self.reverse
        return self._hot

    def col_type(self, reverse):
        if bool(reverse) != self.reverse:
            raise RuntimeError('ReadoutSubgraph was built for reverse=%s' % self.reverse)
        return self._col_type

    def backward_structs(self, reverse, num_types):
        """CSR by SOURCE (N_src keys, compact destination ids as payload) and the relation-grouped edge list."""
        key = ('bwd', int(num_types))
        if key not in self._bwd:
            E2 = self.E
            counts = (self.row_ptr[1:] - self.row_ptr[:-1]).long()
            dst = torch.repeat_interleave(torch.arange(self.N, device=self.device, dtype=torch.int32), counts, output_size=E2)
            src, et = self.col_src[:E2], self.col_type(reverse)[:E2]
            t_row_ptr, t_col_dst, t_col_type, _ = build_csr(src, dst, et, self.N_src)
            rel_ptr, rel_src, rel_dst, _ = build_csr(et, src, dst, num_types)
            self._bwd[key] = (t_row_ptr, t_col_dst, t_col_type, rel_ptr, rel_src, rel_dst)
        return self._bwd[key]


def _to_device(t, device):
    if device.type != 'cuda':
        raise RuntimeError('renet_b200: graphs live on a CUDA device (got %s); no CPU fallback' % device)
    return t.pin_memory().to(device, non_blocking=True) if t.numel() else t.to(device)


def build_csr(key, payload_a, payload_b, n_keys, want_perm=False):
    """Device-side stable grouping by ``key`` (int32 tensors) through renet_build_csr.
    Returns (ptr [n_keys+1], a_sorted, b_sorted, perm or None)."""
    L = _lib.lib()
    _lib.require_cuda(key, payload_a, payload_b)
    E = int(key.numel())
    dev = key.device
    ptr_ = torch.empty(n_keys + 1, dtype=torch.int32, device=dev)
    a = torch.empty(E, dtype=torch.int32, device=dev)
    b = torch.empty(E, dtype=torch.int32, device=dev)
    perm = torch.empty(E, dtype=torch.int32, device=dev) if want_perm else None
    nbytes = int(L.renet_csr_workspace_bytes(n_keys, E))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    rc = L.renet_build_csr(_lib.ptr(key), _lib.ptr(payload_a), _lib.ptr(payload_b), n_keys, E, _lib.ptr(ptr_),
                           _lib.ptr(a), _lib.ptr(b), _lib.ptr(perm), _lib.ptr(ws), nbytes, _lib.stream())
    _lib.check(rc, 'renet_build_csr')
    return ptr_, a, b, perm
