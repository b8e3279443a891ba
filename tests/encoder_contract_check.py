"""The whole RE-Net encoder per query row and per gradient row against float64: the one-call inference encoder
(renet_prepare_sequences + renet_encode_fwd), its fallback and the training path (cases for
tests/test_gpu_encoder_contract.py; importing this module needs no GPU).

What is checked is how the kernels are put together: a batch turned into kernel arguments (sample order, s_idx, read-out
rows, row_glob, sequence starts, the read-out sub-graph, isolation groups), renet_prepare_sequences, renet_encode_fwd with
its phase-1 GRU work forked onto a side stream, and the backward chain fused_gru_backward -> renet_rgcn_bipartite_bwd ->
the self-loop backward through loop_index -> _rows_to_table_grad.  Each kernel family has its own suite.

Reference.  oracle/restate.py in float64 on the device (assemble_batch, batch_graphs, rgcn_block_layer, packed_inputs,
gru_final_hidden_batched): it does not use the package's batchers, and tests/test_oracle_golden.py pins it to the reference
implementation's goldens.  Parameters, norm and the global rows are cast to double.  Gradients come from fp64 autograd of
sum(s_h * G4) + sum(s_q * G3), G4 and G3 fixed random [B, h] matrices (the decoder has its own suite).  A grouped view is
restated group by group, which is what the grouped plan promises.

Row identity.  hb.s_idx must equal the restatement's stable order; every row of s_h / s_q is compared with the restatement's
row of the same sample; rows from Q on (samples without history) must be +0.0 bit for bit; gradient rows that fp64 autograd
leaves at exactly 0 (entities and relations the batch never touches) must be exactly 0.

Bar.  Per row: |got - ref|_inf <= tau (|ref_row|_inf + 1e-2 |ref_tensor|_inf), tau = 1e-4 for s_h and s_q, 5e-4 for the
gradients: each entity and relation row, each relation row of the RGCN weights, each row of the loop weights and the GRU
matrices, each bias vector as a whole.

Discriminating power.  Before any GPU comparison every case applies these mistakes to its float64 restatement and asserts
that each misses the forward bar by at least 10x (MISS): on every targeted row for 1-4, on the worst row for the others.
  swap       two samples of equal history length swap histories (rows with identical histories are never picked)
  comp       a read-out row reads its subject's row in the neighbouring timestamp's component
  glob       a read-out row takes the global row of the neighbouring timestamp
  drop-last  a sequence loses its last step
  col        the entity ids come from the other triplet column (renet_prepare_sequences' col_s)
  rel-half   the relation rows come from the other direction's half of rel_embeds
  norm-full  layer 2 uses the whole timestamp graph's norm instead of the induced sub-graph's
  drop-edge  a layer-1 edge into an in-neighbour (itself not read out) of a read-out node is dropped: two hops out
A mistake the case's batch cannot express (no two sequences of equal length, no edges ...) is reported as n/a; each case
lists the ones it requires.  Grouped cases require col, rel-half and "groups merged" (the batch restated as one group).

Paths.  fast: eval() + no_grad() with a HistoryView, triplets on the device and global-table keys == the graph store's
times; prepare_sequences_kernel must run and, where the split applies (GEMM engine 1, 3h % 200 == 0), the phase-1 kernels
(concat_bias_kernel, the PQ / PT GEMMs) must run on a stream other than the caller's.  fallback: lists (numpy batcher), or a
view whose graph store lacks timestamps of the global table; prepare_sequences_kernel must not run.  train: train(),
dropout 0, RENet.encode then backward.  Which kernels ran is read from torch.profiler traces (the union over up to ten)."""
import contextlib
import copy
import functools
import re

import numpy as np
import torch

from oracle import restate

DEV = 'cuda:0'
TAU_FWD, TAU_GRAD = 1e-4, 5e-4
FLOOR = 1e-2
MISS = 10.0
RGCN_SCALE = 8.0           # the relation weights' scale over the default initialisation (make_model)
WORST = {}                 # (path, output) -> (largest err / bar, case)
MISSES = {}                # mistake -> (smallest miss / bar over the cases, case)
GRAD_KEYS = ['ent_embeds', 'rel_embeds', 'aggregator.rgcn1.weight', 'aggregator.rgcn1.loop_weight', 'aggregator.rgcn2.weight',
             'aggregator.rgcn2.loop_weight'] + ['%s.%s_l0' % (e, w) for e in ('encoder', 'encoder_r')
                                                for w in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')]
ALL_MUTS = ('swap', 'comp', 'glob', 'drop-last', 'col', 'rel-half', 'norm-full', 'drop-edge')


# ---- data ---------------------------------------------------------------------------------------------------------------------
class Data:
    """One batch: triplets [B, 3], per direction the history lists of the batch's samples, the graph dicts (the package's and
    the restatement's PlainGraphs, built from the same quadruples), the global table and optional isolation groups."""

    def __init__(self, quads, num_e, R, h, nb, sel, hists, glob, groups=None, trip=None):
        self.num_e, self.R, self.h, self.nb = num_e, R, h, nb
        self.trip = np.ascontiguousarray(quads[sel, :3] if trip is None else trip, dtype=np.int64)
        self.hist = {rev: ([hists[rev][0][i] for i in sel], [hists[rev][1][i] for i in sel]) for rev in (False, True)}
        self.groups = groups
        self.quads = quads
        self.glob = glob
        self.keys = np.asarray(sorted(glob), dtype=np.int64)

    @functools.cached_property
    def gd_pkg(self):
        from renet_b200 import synthetic
        return synthetic.build_graph_dict(self.quads, self.R)

    @functools.cached_property
    def plain(self):
        return restate.build_graph_dict(self.quads, self.R)

    @functools.cached_property
    def gs(self):
        from renet_b200.hoststore import GraphStore
        return GraphStore(self.gd_pkg)

    def table64(self):
        return torch.stack([self.glob[int(t)].reshape(-1) for t in self.keys]).double().to(DEV)

    def lens(self, rev):
        return np.asarray([len(x) for x in self.hist[rev][0]], dtype=np.int64)

    def view(self, rev, hint=None, partial=False):
        """a HistoryView of the batch; partial: over a graph store of only the timestamps the histories reference, as
        pred_r_topk builds it (then the global table's keys differ from the store's times)"""
        from renet_b200.hoststore import GraphStore, HistoryStore
        hist, hist_t = self.hist[rev]
        gs = self.gs
        if partial:
            gs = GraphStore({t: self.gd_pkg[t] for t in sorted({int(t) for ht in hist_t for t in ht})})
        store = HistoryStore(hist, hist_t, self.trip[:, 2 if rev else 0], gs, dedupe=False, reverse=hint)
        return store.select(np.arange(len(self.trip)), self.groups), gs


@functools.lru_cache(maxsize=3)
def tkg(preset, seed, T, h=200):
    from renet_b200 import synthetic
    return synthetic.SyntheticTKG(preset, seed=seed, num_timestamps=T, h_dim=h)


def tkg_data(preset, seed, T, sel, h=200, nb=100):
    t = tkg(preset, seed, T, h)
    return Data(t.quads, t.num_e, t.num_r, h, nb, np.asarray(sel),
                {False: (t.s_hist, t.s_hist_t), True: (t.o_hist, t.o_hist_t)}, t.global_emb)


def by_length(preset, seed, T, want, rev=False, rng_seed=0):
    """indices into the stream: want = {length: count}; samples drawn at random among those with that history length"""
    t = tkg(preset, seed, T)
    lens = np.asarray([len(x) for x in (t.o_hist if rev else t.s_hist)])
    rng = np.random.default_rng(rng_seed)
    out = [rng.choice(np.flatnonzero(lens == L), n, replace=False) for L, n in want.items()]
    return rng.permutation(np.concatenate(out))


def hand_built(all_edge_free, h=200, seed=3):
    """Entities 0..99 are the batch's, 100..199 their partners: every graph holds x -> 100 + x for each x, so an induced
    sub-graph over batch entities has no edges.  Unless all_edge_free, timestamps 0, 48, 96 also hold the history events
    themselves (components with edges next to edge-free ones)."""
    rng = np.random.default_rng(seed)
    R, n, T = 6, 100, 6
    times = [24 * i for i in range(T)]
    quads = [(x, x % R, n + x, t) for t in times for x in range(n)]
    B = 48
    trip = np.stack((rng.integers(0, n, B), rng.integers(0, R, B), rng.integers(0, n, B)), 1)
    hists = {}
    for rev in (False, True):
        H, HT = [], []
        for i in range(B):
            e = int(trip[i, 2 if rev else 0])
            L = int(rng.integers(0, 6))
            ts = sorted(rng.choice(times, L, replace=False).tolist())
            entry = []
            for t in ts:
                nb_ = rng.choice(np.delete(np.arange(n), e), int(rng.integers(1, 4)), replace=False)
                rr = rng.integers(0, R, len(nb_))
                entry.append(np.stack((rr, nb_), 1).astype(np.int64))
                if not all_edge_free and t % 48 == 0:
                    quads += [(int(o), int(r), e, t) if rev else (e, int(r), int(o), t) for r, o in zip(rr, nb_)]
            H.append(entry)
            HT.append(ts)
        hists[rev] = (H, HT)
    quads = np.asarray(sorted(quads, key=lambda q: q[3]), dtype=np.int64)
    g = torch.Generator().manual_seed(seed)
    glob = {t: 0.1 * torch.randn(1, 1, h, generator=g) for t in times}
    return Data(quads, 2 * n, R, h, 100, np.arange(B), hists, glob, trip=trip)


# ---- float64 restatement ------------------------------------------------------------------------------------------------------
def _t(a):
    return torch.as_tensor(np.asarray(a, dtype=np.int64), device=DEV)


def params64(m):
    return {k: v.detach().double().clone().requires_grad_(True) for k, v in m.named_parameters()}


class Restated:
    pass


def _layer(H, W, Wloop, src, dst, et, norm, relu, nb, loop_mask):
    """restate.rgcn_block_layer, with the self-loop rows scaled by a dropout mask when one is given (RGCN.py:36-37)"""
    if loop_mask is None:
        return restate.rgcn_block_layer(H, W, Wloop, src, dst, et, norm, relu, nb)
    out = restate.rgcn_block_layer(H, W, None, src, dst, et, norm, False, nb) + (H @ Wloop) * loop_mask.double()
    return torch.relu(out) if relu else out


def restate_dir(P, d, rev, mut=(None, None), samples=None, table=None, mask1=None, loop1=None, loop2=None, x4=None, x3=None):
    """s_h, s_q [Q, h] in the restatement's (stable, length-descending) order, plus what the mistakes are picked from.
    mask1 (bool [N, h]): layer 1's ReLU taken as this mask (the kernel's own H1 > 0), so that an element whose
    pre-activation is within rounding of 0 cannot flip the sign of its derivative between fp32 and fp64.
    Dropout masks (scale factors, None: no dropout): loop1 [N, h] and loop2 [N, h] on the self-loop rows of layers 1 and 2
    (only layer 2's read-out rows reach the outputs), x4 [S, 4h] and x3 [S, 3h] on the GRU inputs in sequence-major row
    order"""
    kind, arg = mut
    R, nb = d.R, d.nb
    idx = np.arange(len(d.trip)) if samples is None else np.asarray(samples)
    trip = d.trip[idx]
    hist = [d.hist[rev][0][i] for i in idx]
    hist_t = [d.hist[rev][1][i] for i in idx]
    col = 2 if rev else 0
    bh = restate.assemble_batch(hist, hist_t, trip[:, col])
    g = restate.batch_graphs(bh, d.plain)
    Q = len(bh.seq_len)
    et = g.type_o if rev else g.type_s
    norm = torch.as_tensor(g.norm, device=DEV).double()
    keep = np.ones(len(g.src), dtype=bool)
    if kind == 'drop-edge':
        keep[arg] = False
    H0 = P['ent_embeds'][_t(g.id)]
    H1 = _layer(H0, P['aggregator.rgcn1.weight'], P['aggregator.rgcn1.loop_weight'], _t(g.src[keep]), _t(g.dst[keep]),
                _t(et[keep]), norm, mask1 is None, nb, loop1)
    if mask1 is not None:
        H1 = H1 * mask1.double()
    norm2 = torch.as_tensor(parent_norm(d, bh, g), device=DEV).double() if kind == 'norm-full' else norm
    H2 = _layer(H1, P['aggregator.rgcn2.weight'], P['aggregator.rgcn2.loop_weight'], _t(g.src), _t(g.dst), _t(et), norm2,
                False, nb, loop2)
    seq_len = bh.seq_len.copy()
    starts = np.concatenate(([0], np.cumsum(seq_len)[:-1])).astype(np.int64)
    rows = np.arange(len(g.readout))
    if kind == 'swap':
        a, b = arg
        L = seq_len[a]
        rows[starts[a]:starts[a] + L], rows[starts[b]:starts[b] + L] = rows[starts[b]:starts[b] + L].copy(), rows[starts[a]:starts[a] + L].copy()
    readout = g.readout[rows]
    gidx = np.searchsorted(d.keys, np.asarray(bh.row_time, dtype=np.int64)[rows])
    if kind == 'comp':
        readout[arg[0]] = readout[arg[1]]
    if kind == 'glob':
        gidx[arg] = gidx[arg] + 1 if gidx[arg] + 1 < len(d.keys) else gidx[arg] - 1
    if kind == 'drop-last':
        last = starts[arg] + seq_len[arg] - 1
        readout, gidx = np.delete(readout, last), np.delete(gidx, last)
        seq_len[arg] -= 1
    s_col = (2 - col) if kind == 'col' else col
    s_tem = _t(trip[:, s_col][bh.s_idx])
    r_tem = _t(trip[:, 1][bh.s_idx])
    rel = P['rel_embeds'][R:] if rev != (kind == 'rel-half') else P['rel_embeds'][:R]
    table = d.table64() if table is None else table
    X4, X3, _, _ = restate.packed_inputs(H2, _t(readout), seq_len, s_tem, r_tem, P['ent_embeds'], rel, table[_t(gidx)])
    if x4 is not None:
        X4, X3 = X4 * x4.double(), X3 * x3.double()
    out = Restated()
    out.s_h = restate.gru_final_hidden_batched(X4, seq_len, P['encoder.weight_ih_l0'], P['encoder.weight_hh_l0'],
                                               P['encoder.bias_ih_l0'], P['encoder.bias_hh_l0'])
    out.s_q = restate.gru_final_hidden_batched(X3, seq_len, P['encoder_r.weight_ih_l0'], P['encoder_r.weight_hh_l0'],
                                               P['encoder_r.bias_ih_l0'], P['encoder_r.bias_hh_l0'])
    out.bh, out.g, out.Q, out.starts, out.et = bh, g, Q, starts, et
    out.gidx = gidx
    return out


def parent_norm(d, bh, g):
    """every node's norm in its whole timestamp graph (utils.py:113-117 recomputes it on the induced sub-graph instead)"""
    out, o = [], 0
    for t, n in zip(bh.times, g.comp_sizes):
        pg = d.plain[t]
        out.append(pg.norm[[pg.ids[int(e)] for e in g.id[o:o + n]]])
        o += n
    return np.concatenate(out) if out else np.zeros(0, np.float32)


def reference(P, d, rev, mut=(None, None), merged=False, mask1=None):
    """(s_h, s_q) [Q, h] in the order of the whole batch's stable sort; a grouped batch is restated group by group"""
    table = d.table64()
    if d.groups is None or merged:
        r = restate_dir(P, d, rev, mut, table=table, mask1=mask1)
        return r.s_h, r.s_q, r
    lens = d.lens(rev)
    order = np.argsort(-lens, kind='stable')
    Q = int((lens > 0).sum())
    pos = np.empty(len(lens), dtype=np.int64)
    pos[order] = np.arange(len(lens))
    ids, hs, qs = [], [], []
    for grp in np.unique(d.groups):
        smp = np.flatnonzero(d.groups == grp)
        if lens[smp].sum() == 0:
            continue
        r = restate_dir(P, d, rev, mut, samples=smp, table=table)
        ids.append(smp[r.bh.s_idx[:r.Q]])
        hs.append(r.s_h)
        qs.append(r.s_q)
    where = np.empty(Q, dtype=np.int64)
    where[pos[np.concatenate(ids)]] = np.arange(Q)
    w = _t(where)
    return torch.cat(hs)[w], torch.cat(qs)[w], None


# ---- bars -----------------------------------------------------------------------------------------------------------------------
def row_ratio(got, ref, tau):
    """per row: |got - ref|_inf / (tau (|ref_row|_inf + FLOOR |ref|_inf))"""
    got, ref = got.double().reshape(len(got), -1), ref.double().reshape(len(ref), -1)
    if ref.numel() == 0:
        return torch.zeros(len(ref), dtype=torch.float64, device=ref.device)
    bar = tau * (ref.abs().amax(1) + FLOOR * ref.abs().max())
    err = (got - ref).abs().amax(1)
    return torch.where(bar > 0, err / bar.clamp_min(1e-300), torch.where(err > 0, float('inf'), 0.0).double())


def note(path, what, ratio, case):
    if ratio > WORST.get((path, what), (-1.0,))[0]:
        WORST[(path, what)] = (ratio, case)


def check_forward(case, path, s_h, s_q, ref_h, ref_q):
    Q, B = len(ref_h), len(s_h)
    assert s_h.shape == s_q.shape and B >= Q
    for what, got, ref in (('s_h', s_h, ref_h), ('s_q', s_q, ref_q)):
        assert torch.isfinite(got).all(), (case, path, what, 'not finite')
        tail = got[Q:].contiguous().view(torch.int32)
        assert bool((tail == 0).all()), '%s %s %s: a row from Q = %d on is not +0.0' % (case, path, what, Q)
        r = row_ratio(got[:Q], ref, TAU_FWD)
        worst = float(r.max()) if Q else 0.0
        note(path, what, worst, case)
        assert worst <= 1.0, '%s %s %s: row %d is %.3g x the bar off; %d of %d rows fail' % (
            case, path, what, int(r.argmax()), worst, int((r > 1).sum()), Q)


def check_grads(case, path, got, ref):
    for k in GRAD_KEYS:
        g, r = got[k], ref[k]
        assert g is not None, (case, path, k, 'no gradient')
        g, r = g.reshape(1, -1) if g.dim() == 1 else g, r.reshape(1, -1) if r.dim() == 1 else r
        zero = (r == 0).all(1)
        bad = zero & (g != 0).any(1)
        assert not bool(bad.any()), '%s %s d%s: row %d is exactly 0 in fp64 but not in the kernel\'s gradient' % (
            case, path, k, int(bad.nonzero()[0]))
        ratio = row_ratio(g, r, TAU_GRAD)
        worst = float(ratio.max())
        note(path, 'd' + k, worst, case)
        assert worst <= 1.0, '%s %s d%s: row %d is %.3g x the bar off; %d of %d rows fail' % (
            case, path, k, int(ratio.argmax()), worst, int((ratio > 1).sum()), len(ratio))


# ---- simulated mistakes ----------------------------------------------------------------------------------------------------------
def _miss(mh, mq, ref_h, ref_q, targets, every=True):
    """the smallest (every) or largest row ratio over the targeted rows (None: over all rows)"""
    r = torch.maximum(row_ratio(mh, ref_h, TAU_FWD), row_ratio(mq, ref_q, TAU_FWD))
    r = r if targets is None else r[_t(targets)]
    return float(r.min() if every and targets is not None else r.max())


def candidates(kind, r, d, rev):
    """[(argument, targeted sequence positions or None)] for one mistake, at most 6, most visible first"""
    bh, g, Q, starts = r.bh, r.g, r.Q, r.starts
    L = bh.seq_len
    out = []
    if kind == 'swap':
        for q in range(Q - 1):
            if L[q] == L[q + 1] and not np.array_equal(g.readout[starts[q]:starts[q] + L[q]],
                                                       g.readout[starts[q + 1]:starts[q + 1] + L[q]]):
                out.append(((q, q + 1), [q, q + 1]))
    elif kind == 'comp':
        for q in range(Q):
            if L[q] >= 2:
                k = starts[q] + L[q] - 1
                if g.readout[k] != g.readout[k - 1]:
                    out.append(((k, k - 1), [q]))
    elif kind == 'glob':
        if len(d.keys) > 1:
            out = [(starts[q] + L[q] - 1, [q]) for q in range(Q)]
    elif kind == 'drop-last':
        out = [(q, [q]) for q in range(Q) if L[q] >= 2 and (q + 1 == Q or L[q + 1] < L[q])]
    elif kind == 'col':
        lens = d.lens(rev)
        if np.any(d.trip[lens > 0, 0] != d.trip[lens > 0, 2]):
            out = [(None, None)]
    elif kind == 'rel-half':
        out = [(None, None)]
    elif kind == 'norm-full':
        if not np.array_equal(parent_norm(d, bh, g), g.norm):
            out = [(None, None)]
    elif kind == 'drop-edge':
        ro = set(g.readout.tolist())
        indeg = np.bincount(g.dst, minlength=g.num_nodes)
        by_dst = np.argsort(g.dst, kind='stable')
        ptr = np.concatenate(([0], np.cumsum(indeg)))
        seq_of_row = np.repeat(np.arange(Q), L)
        seqs_of = {}
        for k, v in enumerate(g.readout):
            seqs_of.setdefault(int(v), set()).add(int(seq_of_row[k]))
        last = set(int(g.readout[starts[q] + L[q] - 1]) for q in range(Q))     # read at a sequence's last step: most visible
        for v in sorted((v for v in ro if indeg[v] > 0), key=lambda v: (v not in last, indeg[v])):
            us = set(g.src[by_dst[ptr[v]:ptr[v + 1]]].tolist()) - ro - {v}
            for u in sorted((u for u in us if indeg[u] > 0), key=lambda u: indeg[u])[:2]:
                out.append((int(by_dst[ptr[u]]), sorted(seqs_of[v])))
            if len(out) >= 12:
                break
        return out[:12]
    if kind in ('swap', 'comp', 'glob', 'drop-last') and len(out) > 6:
        pick = np.linspace(0, len(out) - 1, 6).round().astype(int)   # spread over the batch: long and short sequences
        out = [out[i] for i in pick]
    return out[:6]


def discriminate(case, d, P, rev, ref_h, ref_q, r, required):
    """each required mistake must miss the forward bar by MISS x; returns {mistake: miss}"""
    got = {}
    with torch.no_grad():
        if d.groups is not None:
            mh, mq, _ = reference(P, d, rev, merged=True)
            got['merged'] = _miss(mh, mq, ref_h, ref_q, None)
            for kind in ('col', 'rel-half', 'norm-full'):
                mh, mq, _ = reference(P, d, rev, (kind, None))
                got[kind] = _miss(mh, mq, ref_h, ref_q, None)
        else:
            for kind in ALL_MUTS:
                best = None
                for arg, targets in candidates(kind, r, d, rev):
                    m = restate_dir(P, d, rev, (kind, arg))
                    miss = _miss(m.s_h, m.s_q, ref_h, ref_q, targets, kind in ('swap', 'comp', 'glob', 'drop-last'))
                    best = miss if best is None else max(best, miss)
                    if best >= 4 * MISS:
                        break
                if best is not None:
                    got[kind] = best
    for kind in required:
        assert kind in got, '%s: the batch cannot express the mistake %s' % (case, kind)
        assert got[kind] >= MISS, '%s (%s): the mistake %s misses the bar by only %.3g x' % (
            case, 'obj' if rev else 'subj', kind, got[kind])
    for kind, v in got.items():
        if kind in required and v < MISSES.get(kind, (float('inf'),))[0]:
            MISSES[kind] = (v, case)
    return got


# ---- the package's paths ----------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def gemm_engine(engine):
    from renet_b200 import _lib
    if engine is None:
        yield
        return
    before = _lib.lib().renet_set_gemm_engine(engine)
    try:
        yield
    finally:
        _lib.lib().renet_set_gemm_engine(before)


def make_model(d, seed):
    from renet_b200.model import RENet
    torch.manual_seed(seed)
    m = RENet(d.num_e, d.h, d.R, dropout=0, num_bases=d.nb).to(DEV)
    with torch.no_grad():
        # at the default initialisation an edge's message is ~10x smaller than the self-loop term, so a mistake two hops
        # out hides under the bar; scaled relation weights make the graph part of H2 as large as the self-loop part
        for layer in (m.aggregator.rgcn1, m.aggregator.rgcn2):
            layer.weight.mul_(RGCN_SCALE)
    m.global_emb = d.glob
    return m


def encode(m, d, rev, hist, gd, batch=None):
    """RENet.encode of one direction -> (s_h, s_q, hb); hb is what the aggregator built"""
    batch = torch.from_numpy(d.trip).to(DEV) if batch is None else batch
    seen = []
    orig = m.aggregator.encode

    def spy(*a, **k):
        out = orig(*a, **k)
        seen.append(out[2])
        return out
    m.aggregator.encode = spy
    try:
        out = m.encode(batch, None if rev else hist, hist if rev else None, gd, subject=not rev)
    finally:
        del m.aggregator.encode
    return out[3], out[4], seen[0]


def path_inputs(d, rev, path, hint=None):
    if path == 'fallback-lists':
        return d.hist[rev], d.gd_pkg
    return d.view(rev, hint, partial=path == 'fallback-view')


def run_inference(m, d, rev, path, hint=None):
    hist, gd = path_inputs(d, rev, path, hint)
    m.eval()

    def call():
        with torch.no_grad():
            return encode(m, d, rev, hist, gd)
    s_h, s_q, hb = call()
    return s_h, s_q, hb, call


def run_train(m, d, rev, G4, G3, hint=None):
    hist, gd = d.view(rev, hint)
    m.train()
    m.zero_grad(set_to_none=True)
    s_h, s_q, hb = encode(m, d, rev, hist, gd)
    ((s_h * G4).sum() + (s_q * G3).sum()).backward()
    named = dict(m.named_parameters())
    return s_h.detach(), s_q.detach(), hb, {k: (named[k].grad.clone() if named[k].grad is not None else None) for k in GRAD_KEYS}


def trace(fn, done, n=10):
    """{kernel name: set of stream ids} of the kernels fn launches, the union over up to n traces, until done(seen) holds.
    Each trace calls fn twice between two torch kernels, as kernels_of in rgcn_contract_check / support_contract_check do:
    records lost at a trace's edges are the torch kernels', and a kernel that a call launches shows in the second call's
    records even when the first call's were lost, so its absence from a trace means something."""
    prime = torch.zeros(1, device=DEV)
    seen = {}
    for _ in range(n):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            prime.add_(1)
            torch.cuda.synchronize()
            for _ in range(2):
                fn()
                torch.cuda.synchronize()
            prime.add_(1)
            torch.cuda.synchronize()
        for ev in prof.events():
            mm = re.search(r'\b(\w+_kernel)\b', ev.name)
            if mm and ev.device_type == torch.autograd.DeviceType.CUDA:
                seen.setdefault(mm.group(1), set()).add(int(ev.device_resource_id))
        if done(seen):
            break
    return seen


def assert_served(case, path, fn, split):
    """fast: prepare_sequences_kernel ran (on the caller's stream); with the split, concat_bias_kernel and a tensor-core GEMM
    ran off the caller's stream; without it, every GEMM / GRU kernel ran on the caller's stream.
    fallback: prepare_sequences_kernel did not run."""
    def streams(s, prefixes):
        return set().union(*[v for k, v in s.items() if k.startswith(prefixes)])
    gemm = ('umma_gemm', 'sgemm', 'gru_', 'concat_bias', 'pack_transpose')

    if path == 'fast':
        def done(s):
            if 'prepare_sequences_kernel' not in s or not streams(s, gemm):
                return False
            return not split or bool(s.get('concat_bias_kernel', set()) - s['prepare_sequences_kernel'])
        seen = trace(fn, done)
        assert 'prepare_sequences_kernel' in seen, '%s fast: prepare_sequences_kernel did not run (%s)' % (case, sorted(seen))
        main = seen['prepare_sequences_kernel']
        assert len(main) == 1 and streams(seen, ('rgcn_',)) <= main, (case, 'the caller stream is not one stream', seen)
        if split:
            assert seen.get('concat_bias_kernel', set()) and not (seen['concat_bias_kernel'] & main), (
                case, 'phase 1 did not run off the caller stream', seen)
            assert any(k.startswith('umma_gemm') and v - main for k, v in seen.items()), (case, 'no phase-1 GEMM off the caller stream')
        else:
            assert streams(seen, gemm) <= main, (case, 'GRU work off the caller stream without the split', seen)
    else:
        seen = trace(fn, lambda s: bool(streams(s, gemm)))
        assert streams(seen, gemm), (case, 'the trace holds none of the encoder\'s GEMM / GRU kernels', sorted(seen))
        assert 'prepare_sequences_kernel' not in seen, '%s %s: prepare_sequences_kernel ran' % (case, path)


def split_applies(d, engine):
    return (1 if engine is None else engine) == 1 and d.h % 4 == 0 and (3 * d.h) % 200 == 0


def kernel_relu_mask(m, d, rev, hb, r):
    """layer 1's H1 > 0 from the kernels on the package's batch (None for grouped batches, restated group by group).
    This mask is the only way the fp64 gradient reference depends on the kernels' forward: it picks the side of each ReLU
    kink, so that a pre-activation within rounding of 0 cannot put a gradient row off by its whole dout.  The forward checks
    use the unmasked restatement, so a wrong layer-1 forward still fails there."""
    if d.groups is not None:
        return None
    g = hb.graph
    assert np.array_equal(g.node_ent.cpu().numpy(), r.g.id), 'the batchers number the nodes differently'
    with torch.no_grad():
        return m.aggregator.rgcn1.apply_layer(g, m.ent_embeds, g.node_ent, rev) > 0


def _grads64(m, d, rev, mask1, G4, G3):
    """fp64 autograd of sum(s_h G4) + sum(s_q G3) through the restatement"""
    P = params64(m)
    ref_h, ref_q, _ = reference(P, d, rev, mask1=mask1)
    Q = len(ref_h)
    loss = (ref_h * G4[:Q].double()).sum() + (ref_q * G3[:Q].double()).sum()
    keys = [k for k in GRAD_KEYS]
    gr = torch.autograd.grad(loss, [P[k] for k in keys], allow_unused=True)
    return {k: (g if g is not None else torch.zeros_like(P[k])) for k, g in zip(keys, gr)}


def run_case(case, d, paths, dirs=(False, True), required=ALL_MUTS, engine=None, det=False, hint=None, seed=0, rejects=False):
    """every path of the case against one fp64 restatement per direction; rejects: every path must refuse the batch"""
    m = make_model(d, seed)
    P = params64(m)
    B = len(d.trip)
    gen = torch.Generator(device=DEV).manual_seed(seed + 1)
    G4 = torch.randn(B, d.h, device=DEV, generator=gen)
    G3 = torch.randn(B, d.h, device=DEV, generator=gen)
    for rev in dirs:
        tag = '%s-%s' % (case, 'obj' if rev else 'subj')
        lens = d.lens(rev)
        order = np.argsort(-lens, kind='stable')
        with torch.no_grad():
            ref_h, ref_q, r = reference(P, d, rev)
        discriminate(tag, d, P, rev, ref_h, ref_q, r, required)
        with gemm_engine(engine):
            for path in paths:
                if rejects:
                    import pytest
                    with pytest.raises(ValueError, match='history graph has no edge'):
                        if path == 'train':
                            run_train(m, d, rev, G4, G3, hint)
                        else:
                            run_inference(m, d, rev, path, hint)
                    continue
                if path == 'train':
                    ctx = det_mode() if det else contextlib.nullcontext()
                    with ctx:
                        s_h, s_q, hb, grads = run_train(m, d, rev, G4, G3, hint)
                        if det:
                            again = run_train(m, d, rev, G4, G3, hint)[3]
                            for k in GRAD_KEYS:
                                assert torch.equal(grads[k], again[k]), (tag, 'deterministic mode: d%s differs across runs' % k)
                    label = 'train-det' if det else 'train'
                else:
                    s_h, s_q, hb, again = run_inference(m, d, rev, path, hint)
                    label = path
                np.testing.assert_array_equal(np.asarray(hb.s_idx), order, err_msg='%s %s: s_idx' % (tag, path))
                check_forward(tag, label, s_h, s_q, ref_h, ref_q)
                if path == 'train':
                    check_grads(tag, label, grads, _grads64(m, d, rev, kernel_relu_mask(m, d, rev, hb, r), G4, G3))
                else:
                    assert_served(tag, 'fast' if path == 'fast' else path, again, split_applies(d, engine))


@contextlib.contextmanager
def det_mode():
    from rgcn_contract_check import deterministic
    with deterministic(True):
        yield


# ---- the cases ------------------------------------------------------------------------------------------------------------------
CASES = {}


def case(name):
    def reg(fn):
        assert name not in CASES
        CASES[name] = functools.partial(fn, name)
        return fn
    return reg


def bench_data():
    t = tkg('icews18', 999, 240)
    return tkg_data('icews18', 999, 240, t.batch_indices(0, 1024))


@case('bench')
def _(cs):
    """the batch bench.py times: ICEWS18-shaped, 240 timestamps, batch 1024"""
    run_case(cs, bench_data(), ('fast', 'fallback-lists', 'train'))


@case('bench-det')
def _(cs):
    run_case(cs, bench_data(), ('train',), det=True)


@case('gdelt')
def _(cs):
    """many small components"""
    t = tkg('gdelt', 5, 60)
    d = tkg_data('gdelt', 5, 60, t.batch_indices(0, 1024))
    run_case(cs, d, ('fast', 'train'))


@case('q3000')
def _(cs):
    """about 3000 sequences: the persistent recurrence walks a second and a third m-tile of 1152 rows"""
    t = tkg('icews18', 7, 40)
    d = tkg_data('icews18', 7, 40, t.batch_indices(0, 3200))
    assert min(int((d.lens(rev) > 0).sum()) for rev in (False, True)) > 2304
    run_case(cs, d, ('fast', 'train'))


for _rev in (False, True):
    _dir = 'obj' if _rev else 'subj'

    @case('lengths-1-10-' + _dir)
    def _(cs, rev=_rev):
        sel = by_length('icews18', 7, 40, {L: 24 for L in range(1, 11)}, rev, 1)
        run_case(cs, tkg_data('icews18', 7, 40, sel), ('fast', 'fallback-lists', 'train'), dirs=(rev,))

    @case('lengths-all-1-' + _dir)
    def _(cs, rev=_rev):
        sel = by_length('icews18', 7, 40, {1: 200}, rev, 2)
        d = tkg_data('icews18', 7, 40, sel)
        assert set(d.lens(rev)) == {1}
        run_case(cs, d, ('fast', 'fallback-lists', 'train'), dirs=(rev,),
                 required=('swap', 'glob', 'col', 'rel-half', 'norm-full', 'drop-edge'))

    @case('q1-' + _dir)
    def _(cs, rev=_rev):
        t = tkg('icews18', 7, 40)
        hist = t.o_hist if rev else t.s_hist
        # the one sequence: a length-10 history of the fewest neighbours (read-out nodes of small in-degree, so that the
        # two-hop 'drop-edge' shows on the only row there is)
        ten = [i for i in range(len(hist)) if len(hist[i]) == 10]
        one = min(ten, key=lambda i: sum(len(a) for a in hist[i]))
        sel = np.concatenate((by_length('icews18', 7, 40, {0: 40}, rev, 3), [one]))
        d = tkg_data('icews18', 7, 40, sel)
        assert int((d.lens(rev) > 0).sum()) == 1
        run_case(cs, d, ('fast', 'fallback-lists', 'train'), dirs=(rev,),
                 required=('comp', 'glob', 'drop-last', 'col', 'rel-half', 'norm-full', 'drop-edge'))

    @case('trailing-empty-' + _dir)
    def _(cs, rev=_rev):
        want = {0: 150}
        want.update({L: 30 for L in (1, 3, 5, 10)})
        sel = by_length('icews18', 7, 40, want, rev, 4)
        run_case(cs, tkg_data('icews18', 7, 40, sel), ('fast', 'fallback-lists', 'train'), dirs=(rev,))


@case('edge-free-components')
def _(cs):
    d = hand_built(False)
    run_case(cs, d, ('fast', 'fallback-lists', 'train'),
             required=('swap', 'comp', 'glob', 'drop-last', 'col', 'rel-half', 'norm-full'))


@case('edge-free-batch')
def _(cs):
    """E = 0 for the whole batch, which histories drawn from the graph dict never give (DGL would pass h through both
    layers): every path refuses it with a ValueError, the device batcher after waiting for its edge count (the first
    history entry shows no edge on the host)"""
    d = hand_built(True)
    for rev in (False, True):
        hb_E = restate.batch_graphs(restate.assemble_batch(*d.hist[rev], d.trip[:, 2 if rev else 0]), d.plain)
        assert len(hb_E.src) == 0
    # every node's H depends on its entity alone here, so reading another component's row of the subject ('comp') is no
    # mistake the outputs can show
    run_case(cs, d, ('fast', 'fallback-lists', 'train'), required=('swap', 'glob', 'drop-last', 'col', 'rel-half'), rejects=True)


@case('duplicate-subjects')
def _(cs):
    """the same subject twice with different relations (same timestamp: the same history), and the same (s, r) twice"""
    t = tkg('icews18', 7, 40)
    q = t.quads
    late = np.arange(len(q) // 2, len(q))
    key = q[late, 0] * 100000 + q[late, 3]
    _, first, cnt = np.unique(key, return_index=True, return_counts=True)
    pairs = []
    for f in first[cnt >= 2][:60]:
        i = late[f]
        js = late[(q[late, 0] == q[i, 0]) & (q[late, 3] == q[i, 3]) & (q[late, 1] != q[i, 1])]
        if len(js) and len(t.s_hist[i]):
            pairs += [i, int(js[0])]
    pairs = np.asarray(pairs[:80])
    assert len(pairs) >= 40
    sel = np.concatenate((pairs, pairs[:20], t.batch_indices(3, 200)))
    run_case(cs, tkg_data('icews18', 7, 40, sel), ('fast', 'fallback-lists', 'train'))


def grouped_data():
    """as pred_r_topk builds it: one group per entity pair, each repeated once per relation 0..4"""
    t = tkg('icews18', 7, 40)
    q = t.quads
    rng = np.random.default_rng(8)
    late = np.arange(len(q) * 3 // 4, len(q))
    i_s = rng.choice(late[[len(t.s_hist[i]) >= 3 for i in late]], 24, replace=False)
    i_o = rng.choice(late[[len(t.o_hist[i]) >= 3 for i in late]], 24, replace=False)
    R = 5
    n = len(i_s)
    trip = np.stack((np.repeat(q[i_s, 0], R), np.tile(np.arange(R), n), np.repeat(q[i_o, 2], R)), 1)
    hists = {False: ([t.s_hist[i] for i in np.repeat(i_s, R)], [t.s_hist_t[i] for i in np.repeat(i_s, R)]),
             True: ([t.o_hist[i] for i in np.repeat(i_o, R)], [t.o_hist_t[i] for i in np.repeat(i_o, R)])}
    return Data(q, t.num_e, t.num_r, 200, 100, np.arange(n * R), hists, t.global_emb, groups=np.repeat(np.arange(n), R), trip=trip)


@case('grouped-hint')
def _(cs):
    """a HistoryStore with the reverse hint: the read-out sub-graph is built on the loader stream"""
    d = grouped_data()
    for rev in (False, True):
        run_case(cs, d, ('fast', 'train'), dirs=(rev,), required=('merged', 'col', 'rel-half'), hint=rev)


@case('grouped')
def _(cs):
    """without the hint; and over a graph store of only the referenced timestamps (pred_r_topk's): the fallback"""
    run_case(cs, grouped_data(), ('fast', 'fallback-view', 'train'), required=('merged', 'col', 'rel-half'))


@case('engine0')
def _(cs):
    """the FFMA engine: no split, phase 1 returns at once"""
    t = tkg('icews18', 7, 40)
    run_case(cs, tkg_data('icews18', 7, 40, t.batch_indices(1, 512)), ('fast', 'fallback-lists'), engine=0)


def h64_data():
    t = tkg('icews18', 13, 40, 64)
    return tkg_data('icews18', 13, 40, t.batch_indices(0, 512), h=64, nb=8)


@case('h64-nb8')
def _(cs):
    """the generic RGCN kernels (h != 200); 3h % 200 != 0 keeps the GRU unsplit"""
    run_case(cs, h64_data(), ('fast', 'fallback-lists', 'train'))


@case('h64-nb8-det')
def _(cs):
    run_case(cs, h64_data(), ('train',), det=True)


@case('caller-stream')
def _(cs):
    """encode on a non-default stream behind a long kernel and an in-place overwrite of ent_embeds / rel_embeds, all on
    that stream: the fork must wait for the caller's stream (phase 1 reads ent and rel)"""
    t = tkg('icews18', 7, 40)
    d = tkg_data('icews18', 7, 40, t.batch_indices(2, 1024))
    m = make_model(d, 5)
    gen = torch.Generator(device=DEV).manual_seed(6)
    new_ent = torch.randn(m.ent_embeds.shape, device=DEV, generator=gen) * 0.1
    new_rel = torch.randn(m.rel_embeds.shape, device=DEV, generator=gen) * 0.1
    m.eval()
    for rev in (False, True):
        hist, gd = d.view(rev)
        batch = torch.from_numpy(d.trip).to(DEV)
        with torch.no_grad():
            m.ent_embeds.zero_()
            m.rel_embeds.zero_()
            encode(m, d, rev, hist, gd, batch)                 # the old values through the same path first
            side = torch.cuda.Stream(device=DEV)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                torch.cuda._sleep(200_000_000)
                m.ent_embeds.copy_(new_ent)
                m.rel_embeds.copy_(new_rel)
                s_h, s_q, _ = encode(m, d, rev, hist, gd, batch)
            torch.cuda.current_stream().wait_stream(side)
            s_h0, s_q0, _ = encode(m, d, rev, hist, gd, batch)
        P = params64(m)
        ref_h, ref_q, _ = reference(P, d, rev)
        check_forward(cs + ('-obj' if rev else '-subj'), 'fast', s_h, s_q, ref_h.detach(), ref_q.detach())
        assert torch.equal(s_h, s_h0) and torch.equal(s_q, s_q0), (cs, 'the caller-stream result differs from the default stream')


@case('two-devices')
def _(cs):
    """cuda:0, then cuda:1, then cuda:0 in one process, each under torch.cuda.device(i): the side stream and the fork / join
    events are the device's and the caller stream's"""
    import pytest
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    t = tkg('icews18', 7, 40)
    d = tkg_data('icews18', 7, 40, t.batch_indices(4, 512))
    m0 = make_model(d, 9)
    P = params64(m0)
    refs = {rev: reference(P, d, rev)[:2] for rev in (False, True)}
    models = {0: m0.eval()}
    for i in (0, 1, 0):
        dev = torch.device('cuda', i)
        if i not in models:
            from renet_b200 import _lib
            models[i] = copy.deepcopy(m0).to(dev).eval()
            models[i].aggregator._pack_token = _lib.new_pack_token()
            models[i].global_emb = d.glob
        with torch.cuda.device(i):
            for rev in (False, True):
                hist, gd = d.view(rev)
                with torch.no_grad():
                    s_h, s_q, _ = encode(models[i], d, rev, hist, gd, torch.from_numpy(d.trip).to(dev))
                check_forward('%s-cuda%d-%s' % (cs, i, 'obj' if rev else 'subj'), 'fast', s_h.to(DEV), s_q.to(DEV),
                              refs[rev][0].detach(), refs[rev][1].detach())


def summary():
    out = ['%-9s %-28s worst err/bar %.3f  (%s)' % (p, w, v[0], v[1]) for (p, w), v in sorted(WORST.items())]
    out += ['mistake %-10s smallest miss %.1f x the bar  (%s)' % (k, v[0], v[1]) for k, v in sorted(MISSES.items())]
    return out
