"""The whole global model (renet_b200/global_model.py: RENet_global, RGCNAggregator_global) per row against float64 at the
synthetic ICEWS18 and GDELT shapes: the pre-training step's s_q rows, soft targets, loss and every gradient row; the
global-embedding table across its chunks; predict (cases for tests/test_gpu_global_contract.py; importing this module needs
no GPU).

What is checked is how the kernels are put together: whole_graph_arrays (node offsets, type_s / type_o per direction), the
window selection of _windows and get_global_emb, the descending stable sort of t_list and the same permutation of the soft
targets, the zero rows of t == 0, the chunk loop that writes emb[wins], the table's keys (each row keyed by the previous
t), both RGCN layers, the segment pooling, the dense GRU and the soft cross-entropy.  Each kernel family has its own suite.

Reference.  oracle/restate.py (global_windows, global_pooled, global_forward, global_predict, rgcn_block_layer,
gru_final_hidden_batched) in float64 on the device; tests/test_oracle_global.py pins it to the reference implementation's
goldens.  The restatement's graphs are built by oracle/restate.get_big_graph from the same quadruples.  Pooled vectors are
computed once per graph, then the GRU runs over each window (global_predict's definition).  Every case ties the local
composition used for gradients and mistakes to the pinned functions: the pooled rows equal global_pooled's, the loss equals
global_forward's, the table rows equal global_predict's s_q.  Gradients come from float64 autograd of the restated loss.

Row identity.  Each s_q row of a step (recorded by wrapping global_model.decoder_soft_cross_entropy) must match the
restatement's row of the same sorted timestamp, rows of t == 0 must be +0.0 bit for bit and the recorded target rows must
be true_prob[idx] exactly.  get_global_emb must return exactly the restatement's keys in its order, each value [1, 1, h].

Bar.  Per row: |got - ref|_inf <= tau (|ref_row|_inf + 1e-2 |ref_tensor|_inf), tau = 1e-4 for s_q, table and predict rows,
5e-4 for the gradients (each row of ent_embeds, each relation row of the RGCN weights, each row of the loop weights, the
GRU matrices and the linear layer, each bias vector as a whole); the loss within 1e-5 relative.  Gradient rows that fp64
leaves at exactly 0 (entities in no graph of the batch, relations on no edge) must be exactly 0, and the other direction's
linear layer must get no gradient.

Max-pool near-ties.  With ~830 nodes per graph some (graph, column) maxima are within fp32 noise of the runner-up, and the
column's whole gradient goes to whichever node wins.  So the gradient restatement routes each column to the argmax of the
KERNEL's H2 (captured by wrapping _SegmentPoolFn.apply; exact ties to the first node), and separately the kernel-H2 argmax
must equal the fp64 argmax wherever the fp64 gap exceeds GAP relative; the columns inside the gap are counted and printed.
Likewise layer 1's ReLU takes the kernel's H1 > 0 as its mask in the gradient restatement (as the encoder suite does).  The
forward checks use neither.

Discriminating power.  Before any GPU comparison every case applies these mistakes to its float64 restatement and asserts
that each misses the bar by at least MISS: on every targeted row for the first six, on the worst row for the others.
  reverse         the other direction's relation types (type_s <-> type_o)
  window-shift    every window one timestamp later: it includes the query time and drops its oldest graph
  window-short    each window of two or more graphs loses its most recent one
  pool-neighbour  a window's last step takes the pooled row of the neighbouring graph
  target-order    the soft targets taken in t_list order instead of the sorted order (compared as target rows)
  table-key       each table row keyed by its own t instead of the previous one
  pool-mode       mean instead of max, or max instead of mean
  seg-boundary    each graph's last node pooled into the next graph
  layer2-relu     layer 2 gets a ReLU
A mistake a case cannot express is n/a there; each case lists the ones it requires, and every mistake is required by at
least one case.  Max-pool cases cannot show layer2-relu (a column's maximum over hundreds of nodes is positive, so
max(relu(x)) == relu(max(x))) and mean-pool cases cannot show seg-boundary at 10x (one node of ~830 moves the mean by about
4x the bar, the maximum by about 30x); each is required where its pooling mode shows it.

Which kernel ran.  Each case repeats its call under torch.profiler and asserts the RGCN kernels exactly (with template
arguments and the stream kernel's StCfg), and the presence of the deduplicated self-loop kernels, the segment-pool kernels
of the pooling mode, the dense GRU recurrence and the soft-CE epilogues where they apply.

RGCN weights are scaled by RGCN_SCALE over the default initialisation, so that the graph part of H2 is as large as the
self-loop part (otherwise 'reverse' hides under the bar)."""
import contextlib
import functools
import os
import re
import time

import numpy as np
import torch

from oracle import restate

DEV = 'cuda:0'
TAU_FWD, TAU_GRAD = 1e-4, 5e-4
LOSS_TOL = 1e-5
FLOOR = 1e-2
MISS = 10.0
GAP = 1e-5                 # fp64 max-pool gap (relative, with FLOOR) beyond which the kernel must pick the fp64 argmax
RGCN_SCALE = 8.0
SEQ_LEN = 10
H = 200
WORST = {}                 # output -> (largest err / bar, case)
MISSES = {}                # mistake -> (smallest miss / bar over the cases, case)
TIES = {}                  # case -> (columns inside the gap, columns)
GOT = {}                   # case -> {mistake: miss / bar}
GRAD_KEYS = ['ent_embeds', 'aggregator.rgcn1.weight', 'aggregator.rgcn1.loop_weight', 'aggregator.rgcn2.weight',
             'aggregator.rgcn2.loop_weight'] + ['encoder_global.%s_l0' % w for w in ('weight_ih', 'weight_hh', 'bias_ih',
                                                                                     'bias_hh')]
EVERY_ROW = ('reverse', 'window-shift', 'window-short', 'pool-neighbour', 'target-order', 'table-key')
ALL_MUTS = EVERY_ROW + ('pool-mode', 'seg-boundary', 'layer2-relu')
STEP_MUTS = tuple(k for k in ALL_MUTS if k != 'table-key')
TABLE_MUTS = tuple(k for k in ALL_MUTS if k != 'target-order')


# ---- data ---------------------------------------------------------------------------------------------------------------------
class Stream:
    """One synthetic quadruple stream: the package's graph dict, the restatement's PlainGraphs and per-timestamp soft targets
    (each row: the timestamp's subject / object counts, normalised)."""

    def __init__(self, preset, T, seed):
        from renet_b200 import synthetic
        self.quads, self.num_e, self.R = synthetic.make_quads(preset, seed, T)
        self.gd = synthetic.build_graph_dict(self.quads, self.R)
        q = self.quads
        cuts = np.flatnonzero(np.diff(q[:, 3])) + 1
        self.plain = {int(c[0, 3]): restate.get_big_graph(c[:, :3], self.R) for c in np.split(q, cuts)}
        self.times = sorted(self.plain)
        assert list(self.gd) == self.times
        self.unit = self.times[1] - self.times[0]
        self.pos = {t: j for j, t in enumerate(self.times)}
        self.sizes = np.asarray([self.plain[t].number_of_nodes() for t in self.times], dtype=np.int64)
        self.edges = np.asarray([self.plain[t].number_of_edges() for t in self.times], dtype=np.int64)
        ti = np.searchsorted(self.times, q[:, 3])
        self.count_s = np.zeros((len(self.times), self.num_e))
        self.count_o = np.zeros((len(self.times), self.num_e))
        np.add.at(self.count_s, (ti, q[:, 0]), 1.0)
        np.add.at(self.count_o, (ti, q[:, 2]), 1.0)

    def targets(self, sel):
        """(true_prob_s, true_prob_o) [B, num_e] float64 on the device for batch positions of timestamp indices sel"""
        out = []
        for c in (self.count_s, self.count_o):
            rows = c[np.asarray(sel)]
            out.append(torch.from_numpy(rows / rows.sum(1, keepdims=True)).to(DEV))
        return out

    def nodes_of(self, js):
        return int(self.sizes[list(js)].sum())


@functools.lru_cache(maxsize=2)
def stream(preset, T, seed):
    return Stream(preset, T, seed)


def icews18():
    return stream('icews18', 240, 11)


def gdelt():
    return stream('gdelt', 2138, 12)


def _t(a):
    return torch.as_tensor(np.asarray(a, dtype=np.int64), device=DEV)


# ---- float64 restatement ------------------------------------------------------------------------------------------------------
def params64(m):
    return {k: v.detach().double().clone().requires_grad_(True) for k, v in m.named_parameters()}


def layer64(X, W, Wloop, src, dst, et, norm, relu, loop_mask=None, relu_mask=None):
    """restate.rgcn_block_layer with the self-loop rows optionally scaled by a dropout mask and the ReLU optionally taken
    as a fixed mask; with neither it is the same sum in the same order as rgcn_block_layer(..., Wloop, ...)"""
    out = restate.rgcn_block_layer(X, W, None, src, dst, et, norm, False, 100)
    loop = X @ Wloop
    out = out + (loop if loop_mask is None else loop * loop_mask.double())
    if relu_mask is not None:
        return out * relu_mask.double()
    return torch.relu(out) if relu else out


def pooled64(P, s, times, reverse, pool, mut=None, route=None, masks=None, mask1=None):
    """(pooled rows [len(times), h], H2): both layers over the whole graphs of ``times`` batched, then per-graph max / mean.
    route [G, h]: max pooling reads H2 at these absolute rows (the kernel's argmax) instead of taking the max."""
    gs = [s.plain[int(t)] for t in times]
    sizes = np.asarray([g.number_of_nodes() for g in gs], dtype=np.int64)
    off = np.concatenate(([0], np.cumsum(sizes)))
    src = _t(np.concatenate([g.src + o for g, o in zip(gs, off[:-1])]))
    dst = _t(np.concatenate([g.dst + o for g, o in zip(gs, off[:-1])]))
    et = _t(np.concatenate([g.type_o if reverse else g.type_s for g in gs]))
    norm = torch.as_tensor(np.concatenate([g.norm for g in gs]), device=DEV).double()
    H0 = P['ent_embeds'][_t(np.concatenate([g.id for g in gs]))]
    masks = masks or {}
    H1 = layer64(H0, P['aggregator.rgcn1.weight'], P['aggregator.rgcn1.loop_weight'], src, dst, et, norm, True,
                 masks.get('loop1'), mask1)
    H2 = layer64(H1, P['aggregator.rgcn2.weight'], P['aggregator.rgcn2.loop_weight'], src, dst, et, norm,
                 mut == 'layer2-relu', masks.get('loop2'))
    seg = np.repeat(np.arange(len(gs)), sizes)
    if mut == 'seg-boundary':
        seg[off[1:-1] - 1] += 1
    segd = _t(seg)
    cnt = torch.bincount(segd, minlength=len(gs)).double()
    if pool == 1:
        if route is not None:
            return H2.gather(0, route), H2
        out = torch.zeros(len(gs), H2.shape[1], dtype=H2.dtype, device=DEV)
        return out.scatter_reduce(0, segd.view(-1, 1).expand_as(H2), H2, 'amax', include_self=False), H2
    out = torch.zeros(len(gs), H2.shape[1], dtype=H2.dtype, device=DEV).index_add(0, segd, H2)
    return out / cnt.view(-1, 1), H2


def gru64(P, X, lens):
    """final hidden states of windows in any length order (gru_final_hidden_batched wants them sorted descending)"""
    lens = np.asarray(lens, dtype=np.int64)
    order = np.argsort(-lens, kind='stable')
    starts = np.concatenate(([0], np.cumsum(lens)[:-1]))
    rows = np.concatenate([np.arange(starts[q], starts[q] + lens[q]) for q in order])
    h = restate.gru_final_hidden_batched(X[_t(rows)], lens[order], P['encoder_global.weight_ih_l0'],
                                         P['encoder_global.weight_hh_l0'], P['encoder_global.bias_ih_l0'],
                                         P['encoder_global.bias_hh_l0'])
    inv = np.empty_like(order)
    inv[order] = np.arange(len(order))
    return h[_t(inv)]


def window_of(s, q):
    """global_predict's window (Aggregator.py:75-95): indices into s.times of the <= SEQ_LEN graphs before time q"""
    k = sum(1 for t in s.times if t < q)
    return list(range(max(0, k - SEQ_LEN), k))


def mutate_windows(s, wins, mut):
    """(windows, targeted rows) for the window mistakes; windows are lists of indices into s.times"""
    n = len(s.times)
    if mut == 'window-shift':
        tgt = [q for q, w in enumerate(wins) if w and w[-1] + 1 < n]
        return [[j + 1 for j in w] if q in set(tgt) else w for q, w in enumerate(wins)], tgt
    if mut == 'window-short':
        tgt = [q for q, w in enumerate(wins) if len(w) >= 2]
        return [w[:-1] if len(w) >= 2 else w for w in wins], tgt
    if mut == 'pool-neighbour':
        return [w[:-1] + [w[-1] - 1 if w[-1] > 0 else w[-1] + 1] for w in wins], list(range(len(wins)))
    return wins, None


POOL_MUTS = ('reverse', 'pool-mode', 'seg-boundary', 'layer2-relu')


def sq_of_windows(P, s, wins, reverse, pool, mut=None, times=None, route=None, masks=None, mask1=None, pooled=None):
    """s_q [len(wins), h] of windows (index lists into s.times) over the pooled rows of ``times`` (default: every graph);
    pooled: those rows when already computed (a window mistake does not change them)"""
    times = s.times if times is None else times
    at = {s.pos[int(t)]: i for i, t in enumerate(times)}
    pool_m = (1 - pool) if mut == 'pool-mode' else pool
    if pooled is None or mut in POOL_MUTS:
        pooled, _ = pooled64(P, s, times, reverse != (mut == 'reverse'), pool_m, mut, route, masks, mask1)
    X = pooled[_t([at[j] for w in wins for j in w])]
    if masks and 'rows' in masks:
        X = X * masks['rows'].double()
    return gru64(P, X, [len(w) for w in wins])


class Step:
    """one direction of a pre-training step restated: sorted order, windows, targets"""

    def __init__(self, s, t_list, rev):
        self.s, self.rev = s, rev
        self.t = np.asarray(t_list, dtype=np.int64)
        self.idx = np.argsort(-self.t, kind='stable')                                     # global_model.py:45
        wt = restate.global_windows(self.t[self.idx], s.times, SEQ_LEN)                   # Aggregator.py:28-45
        self.wins = [[s.pos[int(t)] for t in w] for w in wt]
        assert self.wins == [window_of(s, int(t)) for t in self.t[self.idx][:len(self.wins)]]
        self.Q = len(self.wins)
        self.uniq = sorted({s.times[j] for w in self.wins for j in w})                   # Aggregator.py:47

    def forward(self, P, pool, tp, mut=None, times=None, route=None, masks=None, mask1=None, pooled=None):
        """(s_q [Q, h], targets [B, num_e], loss) of the restated step"""
        wins, _ = mutate_windows(self.s, self.wins, mut)
        sq = sq_of_windows(P, self.s, wins, self.rev, pool, mut, times, route, masks, mask1, pooled)
        pad = torch.cat((sq, sq.new_zeros(len(self.t) - self.Q, sq.shape[1])), 0)       # global_model.py:51
        lin = 'linear_o' if self.rev else 'linear_s'
        pred = pad @ P[lin + '.weight'].t() + P[lin + '.bias']
        tgt = tp[_t(np.arange(len(self.t)) if mut == 'target-order' else self.idx)]
        return sq, tgt, restate.soft_cross_entropy(pred, tgt)


# ---- bars -----------------------------------------------------------------------------------------------------------------------
def row_ratio(got, ref, tau):
    """per row: |got - ref|_inf / (tau (|ref_row|_inf + FLOOR |ref|_inf))"""
    got, ref = got.double().reshape(len(got), -1), ref.double().reshape(len(ref), -1)
    if ref.numel() == 0:
        return torch.zeros(len(ref), dtype=torch.float64, device=ref.device)
    bar = tau * (ref.abs().amax(1) + FLOOR * ref.abs().max())
    err = (got - ref).abs().amax(1)
    return torch.where(bar > 0, err / bar.clamp_min(1e-300), torch.where(err > 0, float('inf'), 0.0).double())


def note(what, ratio, case):
    if ratio > WORST.get(what, (-1.0,))[0]:
        WORST[what] = (ratio, case)


def check_rows(case, what, got, ref, tau=TAU_FWD):
    assert got.shape == ref.shape, (case, what, tuple(got.shape), tuple(ref.shape))
    assert torch.isfinite(got).all(), (case, what, 'not finite')
    r = row_ratio(got, ref, tau)
    worst = float(r.max()) if len(r) else 0.0
    note(what, worst, case)
    assert worst <= 1.0, '%s %s: row %d is %.3g x the bar off; %d of %d rows fail' % (
        case, what, int(r.argmax()), worst, int((r > 1).sum()), len(r))


def check_grads(case, got, ref):
    for k, r in ref.items():
        g = got[k]
        assert g is not None, (case, k, 'no gradient')
        g, r = (g.reshape(1, -1), r.reshape(1, -1)) if r.dim() == 1 else (g, r)
        bad = (r == 0).all(1) & (g != 0).any(1)
        assert not bool(bad.any()), '%s d%s: row %d is exactly 0 in fp64 but not in the kernel\'s gradient' % (
            case, k, int(bad.nonzero()[0]))
        check_rows(case, 'd' + k, g, r, TAU_GRAD)


# ---- simulated mistakes ----------------------------------------------------------------------------------------------------------
def record_miss(case, got, required, pool=0):
    # max(relu(x)) == relu(max(x)): over hundreds of nodes a column's maximum is positive, so a layer-2 ReLU shows only
    # through a mean pool; and one node moved between graphs of ~830 moves a mean by about 4x the bar, a maximum by 30x
    drop = {1: 'layer2-relu', 0: 'seg-boundary'}[pool]
    required = tuple(k for k in required if k != drop)
    GOT[case] = got
    for kind in required:
        assert kind in got, '%s: the inputs cannot express the mistake %s' % (case, kind)
        assert got[kind] >= MISS, '%s: the mistake %s misses the bar by only %.3g x' % (case, kind, got[kind])
        if got[kind] < MISSES.get(kind, (float('inf'),))[0]:
            MISSES[kind] = (got[kind], case)


def _miss(mq, ref, targets, kind):
    r = row_ratio(mq, ref, TAU_FWD)
    if kind in EVERY_ROW:
        return float(r[_t(targets)].min()) if len(targets) else None
    return float(r.max())


def discriminate_step(case, st, P, pool, tp, ref_sq, ref_tgt, required, pooled):
    got = {}
    with torch.no_grad():
        for kind in STEP_MUTS:
            if kind == 'target-order':
                tgt = [i for i in range(len(st.t)) if st.idx[i] != i and not torch.equal(tp[st.idx[i]], tp[i])]
                if tgt:
                    _, mt, _ = st.forward(P, pool, tp, kind, pooled=pooled)
                    got[kind] = float(row_ratio(mt, ref_tgt, TAU_FWD)[_t(tgt)].min())
                continue
            targets = list(range(st.Q)) if kind in POOL_MUTS else mutate_windows(st.s, st.wins, kind)[1]
            mq, _, _ = st.forward(P, pool, tp, kind, pooled=pooled)
            v = _miss(mq, ref_sq, targets, kind)
            if v is not None:
                got[kind] = v
    record_miss(case, got, required, pool)
    return got


# ---- the package's paths ----------------------------------------------------------------------------------------------------------
def make_model(s, pool, seed, dropout=0.0):
    from renet_b200.global_model import RENet_global
    torch.manual_seed(seed)
    m = RENet_global(s.num_e, H, s.R, dropout=dropout, model=3, seq_len=SEQ_LEN, num_k=10, maxpool=pool).to(DEV)
    with torch.no_grad():
        for layer in (m.aggregator.rgcn1, m.aggregator.rgcn2):
            layer.weight.mul_(RGCN_SCALE)
    return m


class RecordingDropout(torch.nn.Module):
    """nn.Dropout that draws its mask with torch and keeps it (in call order)"""

    def __init__(self, p):
        super().__init__()
        self.p, self.masks = p, []

    def forward(self, x):
        if not self.training or self.p == 0:
            return x
        mask = (torch.rand(x.shape, device=x.device) >= self.p).to(x.dtype) / (1.0 - self.p)
        self.masks.append(mask)
        return x * mask


def swap_dropouts(m):
    """every nn.Dropout of the model -> RecordingDropout; returns {name: module}"""
    out = {}
    for name, mod in list(m.named_modules()):
        for attr, child in list(mod.named_children()):
            if isinstance(child, torch.nn.Dropout):
                rec = RecordingDropout(child.p)
                setattr(mod, attr, rec)
                out[(name + '.' if name else '') + attr] = rec
    return out


@contextlib.contextmanager
def spies(m, budget=None):
    """records what the model computes on its way: the s_q and target rows handed to decoder_soft_cross_entropy, and per
    _global_info call the kernel's H1 and the pooled H2 with its segment offsets"""
    from renet_b200 import global_model as gm
    rec = {'ce': [], 'pool': [], 'h1': []}
    orig_ce, orig_fn, orig_budget = gm.decoder_soft_cross_entropy, gm._SegmentPoolFn, gm.GLOBAL_EMB_NODE_BUDGET

    def ce(s_q, w, b, tp):
        rec['ce'].append((s_q.detach().clone(), tp.detach().clone()))
        return orig_ce(s_q, w, b, tp)

    class Pool:
        @staticmethod
        def apply(H2, seg, mode):
            rec['pool'].append((H2.detach().clone(), seg.detach().cpu().numpy().astype(np.int64), mode))
            return orig_fn.apply(H2, seg, mode)

    layer = m.aggregator.rgcn1
    orig_apply = layer.apply_layer

    def apply_layer(*a, **k):
        out = orig_apply(*a, **k)
        rec['h1'].append(out.detach().clone())
        return out
    gm.decoder_soft_cross_entropy, gm._SegmentPoolFn = ce, Pool
    layer.apply_layer = apply_layer
    if budget is not None:
        gm.GLOBAL_EMB_NODE_BUDGET = budget
    try:
        yield rec
    finally:
        gm.decoder_soft_cross_entropy, gm._SegmentPoolFn, gm.GLOBAL_EMB_NODE_BUDGET = orig_ce, orig_fn, orig_budget
        del layer.apply_layer


@contextlib.contextmanager
def budget_only(budget):
    from renet_b200 import global_model as gm
    before = gm.GLOBAL_EMB_NODE_BUDGET
    gm.GLOBAL_EMB_NODE_BUDGET = before if budget is None else budget
    try:
        yield
    finally:
        gm.GLOBAL_EMB_NODE_BUDGET = before


def seg_argmax(Hm, off):
    """per (segment, column): the first maximum's absolute row, the maximum and the runner-up"""
    G, N, d = len(off) - 1, Hm.shape[0], Hm.shape[1]
    seg = _t(np.repeat(np.arange(G), np.diff(off))).view(-1, 1).expand(N, d)
    mx = torch.zeros(G, d, dtype=Hm.dtype, device=DEV).scatter_reduce(0, seg, Hm, 'amax', include_self=False)
    rows = torch.arange(N, device=DEV).view(-1, 1).expand(N, d)
    cand = torch.where(Hm == mx.gather(0, seg), rows, N)
    arg = torch.full((G, d), N, dtype=torch.long, device=DEV).scatter_reduce(0, seg, cand, 'amin', include_self=True)
    rest = Hm.masked_fill(rows == arg.gather(0, seg), float('-inf'))
    mx2 = torch.full((G, d), float('-inf'), dtype=Hm.dtype, device=DEV).scatter_reduce(0, seg, rest, 'amax', include_self=True)
    return arg, mx, mx2


def check_ties(case, H2k, H2r, off):
    """the kernel-H2 argmax must be the fp64 argmax wherever the fp64 gap is clear; returns the kernel-H2 argmax"""
    arg_k, _, _ = seg_argmax(H2k, off)
    arg_r, mx, mx2 = seg_argmax(H2r, off)
    clear = (mx - mx2) > GAP * (mx.abs() + FLOOR * H2r.abs().max())
    bad = clear & (arg_k != arg_r)
    assert not bool(bad.any()), '%s: the kernel\'s H2 puts %d clear (graph, column) maxima on another node' % (
        case, int(bad.sum()))
    near = int((~clear).sum())
    prev = TIES.get(case, (0, 0))
    TIES[case] = (prev[0] + near, prev[1] + clear.numel())
    return arg_k


# ---- which kernels ran ------------------------------------------------------------------------------------------------------------
def trace(fn, n=10, want=None):
    """the union of the CUDA kernel names over up to n traces of fn (each trace calls fn twice between two torch kernels:
    records lost at a trace's edges are the torch kernels'), until want(names) holds"""
    prime = torch.zeros(1, device=DEV)
    seen = set()
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
        seen |= {ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA}
        if want is None or want(seen):
            break
    return seen


_RGCN_FLAGS = {'rgcn_gather_stream_kernel': 4, 'rgcn_gather_d200_kernel': 3, 'rgcn_dh_tile_kernel': 2, 'rgcn_dw_d200_kernel': 2}


def rgcn_kernels(names):
    """{(kernel, template booleans, StCfg tuple or None)} of the rgcn_* kernels among the names"""
    out = set()
    for nm in names:
        m = re.search(r'rgcn_\w+_kernel', nm)
        if not m or 'kernel' not in nm:
            continue
        tail = nm[m.end():].split('(float', 1)[0].split('(const', 1)[0]
        flags = re.findall(r'true|false|\(bool\)[01]', tail)
        n = _RGCN_FLAGS.get(m.group(0), 0)
        assert len(flags) >= n, nm
        cfg = re.search(r'StCfg<([^>]*)>', nm)
        if cfg:
            args = cfg.group(1).replace('(bool)', '').replace('false', '0').replace('true', '1')
            cfg = tuple(int(x) for x in re.findall(r'\d+', args))
        out.add((m.group(0), tuple(f in ('true', '(bool)1') for f in flags[:n]), cfg))
    return out


HUB_CFG, PLAIN_CFG = (32, 2, 49, 0, 64), (32, 2, 82, 0, 0)


def expected_rgcn(layer1, layer2, dh=None, det=False):
    """layer1 / layer2: 'stream' or 'tile' forward; dh: None (no backward), 'stream' or 'tile'"""
    T, F = True, False
    out = {('rgcn_gather_stream_kernel', (T, T, T, F), HUB_CFG) if layer1 == 'stream' else
           ('rgcn_gather_d200_kernel', (T, T, T), None),
           ('rgcn_gather_stream_kernel', (F, T, F, F), PLAIN_CFG) if layer2 == 'stream' else
           ('rgcn_gather_d200_kernel', (F, T, F), None)}
    if dh is not None:
        out.add(('rgcn_gather_stream_kernel', (F, F, F, T), (32, 2, 77, 1, 0)) if dh == 'stream' else
                ('rgcn_dh_tile_kernel', (F, det), None))
        out |= {('rgcn_dw_d200_kernel', (T, det), None), ('rgcn_dw_d200_kernel', (F, det), None)}
        if det:
            out.add(('rgcn_dw_reduce_kernel', (), None))
    return out


def short_names(names):
    from support_contract_check import short_name
    return {short_name(n) for n in names if 'kernel' in n}


def assert_served(case, fn, rgcn=None, pool=1, dedup=True, backward=False, soft_ce=True):
    def has(names, pattern):
        return any(re.search(pattern, n) for n in names)
    soft = [r'umma_gemm_packed_kernel<(false|\(bool\)0), (\(int\))?3>', r'soft_ce_reduce_kernel']
    if backward:
        soft += [r'umma_gemm_packed_kernel<(false|\(bool\)0), (\(int\))?4>', r'rowsum_accum_kernel']
    want = ['segment_pool_fwd_kernel<%s>' % ('true' if pool == 1 else 'false')]
    if backward:
        want.append('segment_max_bwd_kernel' if pool == 1 else 'segment_mean_bwd_kernel')
    if dedup:
        want += ['dedup_insert_kernel', 'dedup_expand_kernel']

    def done(names):
        sn = short_names(names)
        return (all(w in sn for w in want) and bool(sn & {'gru_recur_kernel', 'gru_gate_kernel'})
                and (not soft_ce or all(has(names, p) for p in soft)) and (rgcn is None or rgcn <= rgcn_kernels(names)))
    names = trace(fn, want=done)
    sn = short_names(names)
    for w in want:
        assert w in sn, '%s: %s did not run (%s)' % (case, w, sorted(sn))
    assert sn & {'gru_recur_kernel', 'gru_gate_kernel'}, '%s: no dense GRU recurrence kernel ran (%s)' % (case, sorted(sn))
    if not dedup:
        assert 'dedup_insert_kernel' not in sn, '%s: the deduplicated self-loop product ran' % case
    if soft_ce:
        for p in soft:
            assert has(names, p), '%s: no kernel matches %s (%s)' % (case, p, sorted(sn))
    if rgcn is not None:
        seen = rgcn_kernels(names)
        assert seen == rgcn, '%s: ran %s, expected %s' % (case, sorted(seen), sorted(rgcn))


# ---- the pre-training step --------------------------------------------------------------------------------------------------------
def run_step(m, s, t_list, tp_s, tp_o, rev, backward=True):
    """RENet_global.forward (+ backward) of one direction on the kernels -> (loss, s_q, targets, grads, rec)"""
    m.zero_grad(set_to_none=True)
    tb = torch.as_tensor(np.asarray(t_list), device=DEV)
    with spies(m) as rec:
        loss = m(tb, tp_s, tp_o, s.gd, subject=not rev)
        if backward:
            loss.backward()
    grads = {k: (p.grad.detach().clone() if p.grad is not None else None) for k, p in m.named_parameters()}
    assert len(rec['ce']) == 1 and len(rec['pool']) == 1 and len(rec['h1']) == 1
    return loss.detach(), rec['ce'][0][0], rec['ce'][0][1], grads, rec


def host_step(case, s, st, want_nodes=None, t0=True, short=True, repeat=True):
    """the properties a step case exists for, on the host"""
    nodes = s.nodes_of([s.pos[t] for t in st.uniq])
    edges = int(s.edges[[s.pos[t] for t in st.uniq]].sum())
    if want_nodes is not None:
        assert want_nodes[0] <= nodes <= want_nodes[1], (case, nodes, want_nodes)
    assert not t0 or (st.t == 0).any(), (case, 'no t == 0')
    assert not short or any(len(w) == 1 for w in st.wins), (case, 'no one-graph window')
    assert not repeat or len(np.unique(st.t)) < len(st.t), (case, 'no repeated timestamp')
    return nodes, edges


def check_step(case, s, sel, pool, dirs=(False, True), det=False, dropout=0.0, hubs_ab=False, required=STEP_MUTS,
               want_nodes=None, kernels=None, seed=0, **host):
    from rgcn_contract_check import deterministic
    m = make_model(s, pool, seed, dropout)
    recs = swap_dropouts(m) if dropout else {}
    m.train()
    t_list = np.asarray([s.times[i] for i in sel], dtype=np.int64)
    tp_s, tp_o = s.targets(sel)
    for rev in dirs:
        tag = '%s-%s' % (case, 'obj' if rev else 'subj')
        tp = tp_s if rev else tp_o
        st = Step(s, t_list, rev)
        host_step(tag, s, st, want_nodes, **host)
        P = params64(m)
        with torch.no_grad():
            pooled_ref = restate.global_pooled(P, s.times, s.plain, rev, pool)
            mine, _ = pooled64(P, s, s.times, rev, pool)
            assert float((mine - pooled_ref).abs().max()) <= 1e-12 * float(pooled_ref.abs().max()), tag
            ref_sq, ref_tgt, loss64 = st.forward(P, pool, tp, pooled=pooled_ref)
            pinned = restate.global_forward(P, t_list, tp_s, tp_o, s.plain, not rev, maxpool=pool)
            assert abs(float(loss64) - float(pinned)) <= 1e-12 * abs(float(pinned)), (tag, float(loss64), float(pinned))
        discriminate_step(tag, st, P, pool, tp, ref_sq, ref_tgt, required, pooled_ref)
        for r in recs.values():
            r.masks.clear()
        ctx = deterministic(True) if det else contextlib.nullcontext()
        with ctx:
            loss, sq, tgt, grads, rec = run_step(m, s, t_list, tp_s, tp_o, rev)
            if det:
                again = run_step(m, s, t_list, tp_s, tp_o, rev)
                assert torch.equal(again[0], loss) and torch.equal(again[1], sq), (tag, 'deterministic mode: s_q differs')
                for k, g in grads.items():
                    assert (g is None and again[3][k] is None) or torch.equal(g, again[3][k]), (tag, 'deterministic: d' + k)
        # ---- forward
        masks = None
        if dropout:
            assert [len(recs[k].masks) for k in ('aggregator.rgcn1.dropout', 'aggregator.rgcn2.dropout', 'aggregator.dropout')] \
                == [1, 1, 1], (tag, {k: len(r.masks) for k, r in recs.items()})
            masks = {'loop1': recs['aggregator.rgcn1.dropout'].masks[0], 'loop2': recs['aggregator.rgcn2.dropout'].masks[0],
                     'rows': recs['aggregator.dropout'].masks[0]}
            with torch.no_grad():
                ref_sq, ref_tgt, loss64 = st.forward(P, pool, tp, times=st.uniq, masks=masks)
        assert sq.shape == (len(t_list), H) and torch.equal(tgt, ref_tgt), (tag, 'target rows are not true_prob[idx]')
        assert bool((sq[st.Q:].contiguous().view(torch.int32) == 0).all()), (tag, 'a row of t == 0 is not +0.0')
        check_rows(tag, 's_q', sq[:st.Q], ref_sq)
        lerr = abs(float(loss) - float(loss64)) / abs(float(loss64))
        note('loss (rel err / 1e-5)', lerr / LOSS_TOL, tag)
        assert lerr <= LOSS_TOL, (tag, 'loss', float(loss), float(loss64))
        # ---- gradients: routed through the kernel's argmax and ReLU side
        H2k, off, _ = rec['pool'][0]
        gs = [s.gd[t] for t in st.uniq]
        assert np.array_equal(np.concatenate([g.node_id for g in gs]),
                              np.concatenate([s.plain[t].id for t in st.uniq])), 'the graphs number their nodes differently'
        assert np.array_equal(off, np.concatenate(([0], np.cumsum([s.plain[t].number_of_nodes() for t in st.uniq])))), tag
        route = None
        if pool == 1:
            with torch.no_grad():
                _, H2r = pooled64(P, s, st.uniq, rev, pool, masks=masks)
            route = check_ties(tag, H2k.double(), H2r, off)
        mask1 = rec['h1'][0] > 0
        _, _, lg = st.forward(P, pool, tp, times=st.uniq, route=route, masks=masks, mask1=mask1)
        keys = GRAD_KEYS + ['linear_o.weight', 'linear_o.bias'] if rev else GRAD_KEYS + ['linear_s.weight', 'linear_s.bias']
        ref = dict(zip(keys, torch.autograd.grad(lg, [P[k] for k in keys], allow_unused=True)))
        ref = {k: (g if g is not None else torch.zeros_like(P[k])) for k, g in ref.items()}
        other = 'linear_s' if rev else 'linear_o'
        assert grads[other + '.weight'] is None and grads[other + '.bias'] is None, (tag, 'the other direction\'s linear layer')
        check_grads(tag, grads, ref)
        # ---- hub rows on and off
        if hubs_ab:
            os.environ['RENET_STREAM_CFG'] = '3'
            try:
                assert rgcn_kernels(trace(lambda: run_step(m, s, t_list, tp_s, tp_o, rev, False))) >= \
                    {('rgcn_gather_stream_kernel', (True, True, True, False), (32, 2, 82, 0, 0))}, tag
                off_sq = run_step(m, s, t_list, tp_s, tp_o, rev, backward=False)[1]
            finally:
                del os.environ['RENET_STREAM_CFG']
            assert torch.equal(off_sq, sq), (tag, 'hub rows on and off differ')
        if kernels is not None and not dropout:
            ctx = deterministic(True) if det else contextlib.nullcontext()
            with ctx:
                assert_served(tag, lambda: run_step(m, s, t_list, tp_s, tp_o, rev), kernels, pool, dedup=True, backward=True)


# ---- the table and predict --------------------------------------------------------------------------------------------------------
def table_queries(s, t_list):
    """the reference's keys and query times (global_model.py:57-73): each key is the previous t, the last one t_list[-1]"""
    keys, queries, prev = [], [], 0
    for t in t_list:
        if t == 0:
            continue
        keys.append(prev)
        queries.append(t)
        prev = t
    keys.append(t_list[-1])
    queries.append(t_list[-1] + s.unit)
    return keys, queries


def chunks_of(s, wins, budget):
    """the instance-node counts of the chunks get_global_emb's loop makes: windows by length descending, greedily up to
    the node budget"""
    lens = np.asarray([len(w) for w in wins])
    order = np.argsort(-lens, kind='stable')
    nodes = [s.nodes_of(w) for w in wins]
    out, lo = [], 0
    while lo < len(order):
        hi, tot = lo + 1, nodes[order[lo]]
        while hi < len(order) and tot + nodes[order[hi]] <= budget:
            tot += nodes[order[hi]]
            hi += 1
        out.append(tot)
        lo = hi
    return out


def discriminate_windows(case, s, P, wins, pool, reverse, ref, required, pooled, shifted_keys=False):
    got = {}
    with torch.no_grad():
        for kind in ALL_MUTS:
            if kind == 'target-order':
                continue
            if kind == 'table-key':
                if shifted_keys and len(wins) > 1:
                    got[kind] = float(row_ratio(ref[:-1], ref[1:], TAU_FWD).min())     # row i holds row i - 1's value
                continue
            wm, targets = mutate_windows(s, wins, kind)
            if targets is None:
                targets = list(range(len(wins)))
            if kind in EVERY_ROW and not targets:
                continue
            v = _miss(sq_of_windows(P, s, wm, reverse, pool, kind, pooled=pooled), ref, targets, kind)
            if v is not None:
                got[kind] = v
    record_miss(case, got, required, pool)


def check_table(case, s, pool=1, budget=None, min_chunks=2, kernels=None, dedup=True, required=TABLE_MUTS, seed=0,
                chunk_nodes=None):
    from renet_b200 import global_model as gm
    m = make_model(s, pool, seed).eval()
    t_list = list(s.times)
    keys, queries = table_queries(s, t_list)
    wins = [window_of(s, q) for q in queries]
    assert all(wins), (case, 'an empty window')
    chunks = chunks_of(s, wins, gm.GLOBAL_EMB_NODE_BUDGET if budget is None else budget)
    n_chunks, inst = len(chunks), sum(chunks)
    assert n_chunks >= min_chunks, (case, n_chunks, inst)
    assert chunk_nodes is None or chunk_nodes[0] <= min(chunks) and max(chunks) <= chunk_nodes[1], (case, chunks)
    lens = [len(w) for w in wins]
    assert min(lens) == 1 and max(lens) == SEQ_LEN, (case, 'no short window')
    P = params64(m)
    with torch.no_grad():
        pinned = restate.global_pooled(P, s.times, s.plain, False, pool)
        assert float((pooled64(P, s, s.times, False, pool)[0] - pinned).abs().max()) <= 1e-12 * float(pinned.abs().max())
        ref = sq_of_windows(P, s, wins, False, pool, pooled=pinned)
        for q in sorted({0, 1, len(queries) // 2, len(queries) - 1}):
            sq_p, _ = restate.global_predict(P, queries[q], s.plain, True, maxpool=pool)
            assert float((sq_p - ref[q]).abs().max()) <= 1e-10 * float(ref[q].abs().max()), (case, q)
    discriminate_windows(case, s, P, wins, pool, False, ref, required, pinned, shifted_keys=True)
    with spies(m, budget) as rec:
        table = m.get_global_emb(t_list, s.gd)
    assert len(rec['pool']) == n_chunks, (case, 'chunks', len(rec['pool']), n_chunks)
    assert list(table) == keys, (case, 'keys')
    for k in keys:
        assert table[k].shape == (1, 1, H) and not table[k].requires_grad, (case, k)
    check_rows(case, 'table', torch.cat([table[k].view(1, H) for k in keys]), ref)
    if kernels is not None:
        with budget_only(budget):
            assert_served(case, lambda: m.get_global_emb(t_list, s.gd), kernels, pool, dedup=dedup, soft_ce=False)
    return inst, n_chunks


# ---- the cases ------------------------------------------------------------------------------------------------------------------
CASES = {}
SECONDS = {}


def case(name):
    def reg(fn):
        assert name not in CASES

        def run():
            t0 = time.perf_counter()
            fn(name)
            SECONDS[name] = time.perf_counter() - t0
        CASES[name] = run
        return fn
    return reg


def stream_batch():
    """36 unique graphs (about 30 k nodes): t = 0, a one-graph window (t = 24), a repeated timestamp, both orders"""
    return [60, 0, 1, 150, 5, 200, 61, 1]


@case('icews18-step-stream')
def _(cs):
    """layer 1 on the stream kernel with hub rows, layer 2 stream plain, stream dH; hub rows on and off bitwise equal"""
    check_step(cs, icews18(), stream_batch(), 1, hubs_ab=True, want_nodes=(16384, 40960),
               kernels=expected_rgcn('stream', 'stream', 'stream'))


def whole_batch(s, seed):
    return np.random.default_rng(seed).permutation(len(s.times))


@case('icews18-step-tile')
def _(cs):
    """one pre-training batch of all 240 timestamps: tile forward and dH at about 200 k nodes, dW over about 760 k edges,
    the deduplicated self-loop product at about 200 k rows, hub-target scatter into ent_embeds"""
    s = icews18()
    check_step(cs, s, whole_batch(s, 1), 1, want_nodes=(150_000, 250_000), kernels=expected_rgcn('tile', 'tile', 'tile'),
               repeat=False)


@case('icews18-step-tile-mean')
def _(cs):
    s = icews18()
    check_step(cs, s, whole_batch(s, 2), 0, want_nodes=(150_000, 250_000), kernels=expected_rgcn('tile', 'tile', 'tile'),
               repeat=False)


@case('icews18-step-det')
def _(cs):
    """as icews18-step-tile under torch.use_deterministic_algorithms(True): deterministic dH / dW / scatter, two runs bitwise
    equal"""
    s = icews18()
    check_step(cs, s, whole_batch(s, 3), 1, det=True, want_nodes=(150_000, 250_000),
               kernels=expected_rgcn('tile', 'tile', 'tile', det=True), repeat=False)


@case('gdelt-step')
def _(cs):
    """GDELT shape, 2 138 timestamps, a batch of 1 024 consecutive ones (shuffled): tile paths at about 420 k nodes, R2 = 480"""
    s = gdelt()
    sel = 1000 + np.random.default_rng(4).permutation(1024)
    assert 2 * s.R == 480
    check_step(cs, s, sel, 1, want_nodes=(300_000, 600_000), kernels=expected_rgcn('tile', 'tile', 'tile'),
               t0=False, short=False, repeat=False, required=STEP_MUTS)


@case('icews18-table')
def _(cs):
    """get_global_emb over all 240 timestamps, eval, default budget: 2 chunks of about 1 M instance nodes (tile gather at
    N near 10^6, the deduplicated self-loop product at about 1 M rows)"""
    inst, n = check_table(cs, icews18(), kernels=expected_rgcn('tile', 'tile'))
    assert inst > 1_500_000 and n == 2, (inst, n)


@case('icews18-table-small-budget')
def _(cs):
    """GLOBAL_EMB_NODE_BUDGET of about 30 graphs: dozens of chunks of about three windows, windows of equal length split
    across chunks, the mean pool"""
    s = icews18()
    budget = int(30 * s.sizes.mean())
    inst, n = check_table(cs, s, pool=0, budget=budget, min_chunks=40, required=TABLE_MUTS)
    assert n >= 40, n


@case('gdelt-table')
def _(cs):
    """get_global_emb at the GDELT shape: about 8.6 M instance nodes in about 9 chunks"""
    inst, n = check_table(cs, gdelt(), min_chunks=6, kernels=expected_rgcn('tile', 'tile'))
    assert inst > 6_000_000, inst


@case('predict')
def _(cs):
    """RENet_global.predict at several t, both directions: one-graph windows (t = times[1]), short and full windows, and
    the time after the last graph; s_q and the logits of the nn.Linear head"""
    s = icews18()
    m = make_model(s, 1, 5).eval()
    P = params64(m)
    qs = [s.times[1], s.times[2], s.times[7], s.times[120], s.times[-1] + s.unit]
    assert len(window_of(s, qs[0])) == 1 and len(window_of(s, qs[-1])) == SEQ_LEN
    for rev in (False, True):
        tag = '%s-%s' % (cs, 'obj' if rev else 'subj')
        with torch.no_grad():
            refs = [restate.global_predict(P, q, s.plain, not rev) for q in qs]
            ref_sq = torch.stack([r[0] for r in refs])
            wins = [window_of(s, q) for q in qs]
            pooled = restate.global_pooled(P, s.times, s.plain, rev, 1)
            mine = sq_of_windows(P, s, wins, rev, 1, pooled=pooled)
            assert float((mine - ref_sq).abs().max()) <= 1e-10 * float(ref_sq.abs().max()), tag
        discriminate_windows(tag, s, P, wins, 1, rev, ref_sq,
                             ('reverse', 'window-short', 'pool-neighbour', 'pool-mode', 'layer2-relu'), pooled)
        got = []
        with torch.no_grad():
            for q in qs:
                sq, logits, prob = m.predict(q, s.gd, subject=not rev)
                assert sq.shape == (1, 1, H) and logits.shape == (1, 1, s.num_e) and prob.shape == (s.num_e,)
                got.append((sq.view(-1), logits.view(-1)))
        check_rows(tag, 'predict s_q', torch.stack([g[0] for g in got]), ref_sq)
        check_rows(tag, 'predict logits', torch.stack([g[1] for g in got]), torch.stack([r[1] for r in refs]))
    assert_served(cs, lambda: m.predict(qs[0], s.gd), expected_rgcn('tile', 'tile'), 1, dedup=False, soft_ce=False)


@case('train-dropout')
def _(cs):
    """icews18-step-stream in train mode with p = 0.5 (the pre-training configuration): every nn.Dropout records the mask it
    draws, and the restatement applies them to the self-loop rows of both layers and to the GRU input rows.  The mistakes
    are shown on the same batch without dropout."""
    check_step(cs, icews18(), stream_batch(), 1, dropout=0.5, want_nodes=(16384, 40960),
               required=('reverse', 'window-shift', 'window-short', 'pool-neighbour', 'target-order'))


def summary():
    out = ['%-24s worst err/bar %.3f  (%s)' % (w, v[0], v[1]) for w, v in sorted(WORST.items())]
    out += ['mistake %-15s smallest miss %.3g x the bar  (%s)' % (k, v[0], v[1]) for k, v in sorted(MISSES.items())]
    out += ['near-tie columns %-30s %d of %d' % (k, v[0], v[1]) for k, v in sorted(TIES.items())]
    out += ['%-28s %.1f s' % (k, v) for k, v in sorted(SECONDS.items())]
    return out
