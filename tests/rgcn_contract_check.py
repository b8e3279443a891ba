"""The RGCN gather kernels and the layer's backward, per row against float64, on every kernel path, with the serving kernel
asserted (cases for tests/test_gpu_rgcn_contract.py; importing this module needs no GPU).

Reference.  A plain float64 restatement on the device (chunked index_add_) of
  forward   Hout[v] = act(norm[v] * sum_e blockdiag(W[type_e]) . X[src_e] + loop[v])
  backward  P = dHout * [Hout > 0] (from the KERNEL's Hout, so a ReLU sign flip cannot enter),
            dH[u] = sum_{e: src = u} blockdiag(W[type_e])^T . (norm[dst_e] P[dst_e]) + (P @ Wloop^T)[u],
            dW[r] += sum_{e: type = r} X[src_e] (x) norm[dst_e] P[dst_e],  dWloop += X^T @ P
and, beside every reference value, the same sum over absolute values S = sum |term| (|loop row| and |base| included).
The self-loop parts (loop rows, P @ Wloop^T) are dense products of the GEMM engine, which has its own suite
(tests/gemm_contract_check.py): they are taken from renet_selfloop_gemm[_bwd] on the same operands, so what is compared
here is the gather.  dW and dWloop start from a random non-zero base, as in gpu_helpers.layer_bwd.

Bar.  A row passes when |got - ref| <= C * 2^-24 * (n + 4) * S for each of its 200 (dW: 400) elements, n = the row's
in-degree (forward), out-degree (dH) or the relation's edge count (dW).  (n + 4) * 2^-24 * S is the first-order worst case
of an fp32 sum of that many products in any order plus the scale, self-loop and base roundings, so C = 1 holds by
construction; the largest ratio err / ((n + 4) 2^-24 S) seen over all cases on an H100 (80 GB HBM3, 700 W limit) was 0.62
(stream dH 0.62, stream forward 0.55, dW 0.55 in both modes, tile dH 0.53, deterministic tile dH 0.49, tile forward 0.49; every
one on a row with 1 to 3 edges).  A row scaled by 1.0001 is 1678 * 2^-24 of its value off: far outside the bar on
rows of a few edges.  Rows without
edges must equal act(self-loop row), 0 or the base bit for bit, and rows past N must come back untouched.  A failure names
the worst row and its n.

Which kernel ran.  Every case states the kernel it expects; the call is repeated under torch.profiler (CUDA activities, a
call of its own) and the demangled kernel names, template arguments included, must be exactly the expected ones:
rgcn_gather_stream_kernel<RELU, HAS_LOOP, INDEXED, BWD>, rgcn_gather_d200_kernel<RELU, HAS_LOOP, INDEXED>,
rgcn_dh_tile_kernel<HAS_LOOP, DET>, rgcn_dw_d200_kernel<INDEXED, DET> (+ rgcn_dw_reduce_kernel when DET).

Graphs are built from explicit degree sequences / per-relation edge counts, and each case asserts the property it exists
for on the host (with the partition model of tests/test_stream_partition.py) before it launches.  d = 200, 100 blocks.

Cases (id: the branch it exists for)
 stream kernel (rgcn_stream.cuh), forward through renet_rgcn_gather[_hot] / renet_rgcn_block_fwd, dH through
 renet_rgcn_block_bwd:
  rp-global-{fwd,fwd-indexed,bwd}: N = 40 000, the first half carries 260 k edges, the second half one edge at every 8th
      row: CTAs own > 1023 rows and read row_ptr from global memory (rp_in_smem == false)
  hub-{mid,first,last}-{fwd,bwd}: a 6 000-edge row, heavier than a CTA's share (a chain of heads through most warps of one
      CTA, CTA boundary rounding around it); 7 leading and 9 trailing rows without edges; the hub as the first / last row
      that has edges
  r2-<R2>-<uniform|zipf>-{fwd,bwd}: R2 = 1, 40 (all relations resident, empty hot groups), 82 / 77 (= kHot), 83 / 78,
      512, 2048 (the whole slot table), 2049 (use_hot == false: every relation row from L2)
  hist-{saturated,exact}-{fwd,bwd}: a 25 k-edge row over 90 relations (> kHot relations with >= 255 edges in one CTA: the
      threshold stays 256, every slot comes from the "one below the threshold" pass) and over exactly kHot relations
  hot-lists: renet_rgcn_gather_hot with lists of length 0 (non-null pointer), 1, 82, 83, 200, with ids -1 and R2 mixed in,
      with duplicates: torch.equal to the list-free result
  inst-stream-fwd-<r><l><i>: the eight RELU x HAS_LOOP x INDEXED instantiations (HAS_LOOP through renet_rgcn_block_fwd);
      inst-stream-bwd-loop<l>: both backward instantiations; indexed rows repeat heavily in a 23 033-row table
  edge-*: the selection boundaries, expected kernel asserted on each side: N = 2047 / 2048 (plain), 16383 / 16384 (indexed
      forward, backward), 40960 / 40961, E = 16383 / 16384, and a forward launch with E passed as 4x the true count (a
      5 000-edge graph that only the capacity puts on the stream kernel)
  readout-{fwd,bwd,bwd-det}: layer 2 at production shape on a sub-graph built by ReadoutSubgraph (34 000 sources, 8 000
      compact destinations, ~ 95 k edges, launched with the parent's capacity); renet_rgcn_bipartite_bwd in both modes
 tile kernels (rgcn_tile.cuh: rgcn_gather_d200_kernel, rgcn_dh_tile_kernel atomic and DET):
  tile-n<N>-{fwd,bwd,bwd-det}: N = 1, 15, 16, 17, 33 (partial and single tiles)
  tile-span8-*: a row whose edges lie in all 8 warps' slices (seven head slots); tile-hole-*: a tile of 16 rows without
      edges between two full ones; tile-e0-{plain,indexed}: the E = 0 pass-through
  inst-tile-fwd-<r><l><i>, inst-tile-bwd-loop<l>[-det]: every instantiation on a 1 500-row graph
  deterministic dH / dW must be torch.equal across two runs
 dW (rgcn_dw_d200_kernel, default and deterministic, indexed and plain; relation-grouped lists from explicit counts):
  dw-empties: relations without edges first, last and in runs of several between non-empty ones
  dw-run-edges: relation boundaries exactly on multiples of 64 and one edge either side (a relation whose last run holds
      exactly one of its edges, one whose first run does)
  dw-singles-hub: relations with exactly 1 edge next to one with 60 % of the edges
  dw-64-singles: 64 single-edge relations filling one run exactly, between two others
  dw-e<E> (E = 1, 63, 64, 65) and dw-r2-1

Not covered: the generic (non-200) kernels (golden cases only), RENET_GATHER_KERNEL / RENET_STREAM_CFG overrides, and
graphs beyond 2^24 rows (the partition's fourth search round)."""
import contextlib
import functools
import re

import numpy as np
import torch

from test_stream_partition import GRID, NODE_COST, WARPS, cta_boundary, warp_ranges

DEV = 'cuda:0'
EXTRA = 8                  # rows past N in every written buffer: must come back bit for bit
ENT_ROWS = 23033           # ICEWS18 entities: the table indexed inputs gather from
U = 2.0 ** -24
C = 1.0                    # the bar, in units of (n + 4) 2^-24 S; observed: at most 0.62 (module docstring)
K_HOT = {False: 82, True: 77}
RP_CAP = 1024
WORST = {}                 # kernel label -> (largest err / ((n + 4) 2^-24 S), case, what, row, n)


# ---- graphs ------------------------------------------------------------------------------------------------------------------
class Graph:
    """COO edge list kept in destination order (the forward CSR's order)."""

    def __init__(self, n_src, n_dst, R2, src, dst, et, norm=None):
        o = np.argsort(dst, kind='stable')
        self.n_src, self.n_dst, self.R2 = int(n_src), int(n_dst), int(R2)
        self.src, self.dst, self.et = (np.asarray(a, dtype=np.int64)[o] for a in (src, dst, et))
        self.E = len(self.src)
        self.norm = norm

    def ptr(self, key, n):
        return np.concatenate(([0], np.cumsum(np.bincount(key, minlength=n)))).astype(np.int64)

    @property
    def rp_dst(self):
        return self.ptr(self.dst, self.n_dst)

    @property
    def rp_src(self):
        return self.ptr(self.src, self.n_src)


def rel_draw(rng, E, R2, how):
    return rng.integers(0, R2, E) if how == 'uniform' else (rng.zipf(1.3, E) - 1) % R2


def graph_by_degrees(deg, n_other, R2, seed, rel='uniform', by='dst', hub=None, hub_rels=0):
    """deg: the in-degrees (by = 'dst') or out-degrees (by = 'src') of every row; the other endpoint and the relation are
    drawn.  hub / hub_rels: that row's edges cycle through relations 0 .. hub_rels - 1."""
    rng = np.random.default_rng(seed)
    deg = np.asarray(deg, dtype=np.int64)
    key = np.repeat(np.arange(len(deg)), deg)
    other = rng.integers(0, n_other, len(key))
    et = rel_draw(rng, len(key), R2, rel)
    if hub_rels:
        at = np.flatnonzero(key == hub)
        et[at] = np.arange(len(at)) % hub_rels
    if by == 'dst':
        return Graph(n_other, len(deg), R2, other, key, et)
    return Graph(len(deg), n_other, R2, key, other, et)


def graph_by_relations(counts, N, seed):
    rng = np.random.default_rng(seed)
    et = np.repeat(np.arange(len(counts)), counts)
    return Graph(N, N, len(counts), rng.integers(0, N, len(et)), rng.integers(0, N, len(et)), et)


def exact_degrees(N, E, seed):
    """N degrees that sum to exactly E (a uniform draw of E endpoints)"""
    return np.bincount(np.random.default_rng(seed).integers(0, N, E), minlength=N)


@functools.lru_cache(maxsize=4)
def mid_degrees(N=20000):
    """the mid-size graph of most cases: ~ 100 k edges, 7 leading and 9 trailing rows without edges"""
    deg = np.random.default_rng(N).integers(0, 11, N)
    deg[:7] = 0
    deg[-9:] = 0
    return deg


def ctas(rp):
    """[(A, A_next, cb, ce)] of the 132 CTAs by the host partition model"""
    N, E = len(rp) - 1, int(rp[-1])
    b = [cta_boundary(rp, N, E, c) for c in range(GRID + 1)]
    return [(b[c][0], b[c + 1][0], b[c][1], b[c + 1][1]) for c in range(GRID)]


def assert_rp_from_global(rp):
    big = [(a, an, cb, ce) for a, an, cb, ce in ctas(rp) if an - a + 1 > RP_CAP and ce > cb]
    assert big, 'no CTA owns more than %d rows and an edge' % (RP_CAP - 1)


def assert_hub(rp, hub, first=False, last=False):
    deg = np.diff(rp)
    share = (int(rp[-1]) + NODE_COST * (len(rp) - 1)) / GRID
    assert deg[hub] > 4 * share
    with_edges = np.flatnonzero(deg)
    assert deg[0] == 0 and deg[-1] == 0
    assert not first or with_edges[0] == hub
    assert not last or with_edges[-1] == hub
    own = [c for c in ctas(rp) if c[0] <= hub < c[1]]
    assert len(own) == 1
    a, an, cb, ce = own[0]
    e0 = warp_ranges(rp, a, an, cb, ce)
    on_hub = sum(1 for w in range(WARPS) if e0[w] < e0[w + 1] and e0[w] < rp[hub + 1] and e0[w + 1] > rp[hub])
    assert on_hub >= 24, on_hub                    # a chain of heads through (nearly) every warp of the CTA


def assert_histogram(g, bwd, hub, n_rels, saturated):
    key, rp = (g.src, g.rp_src) if bwd else (g.dst, g.rp_dst)
    own = [c for c in ctas(rp) if c[0] <= hub < c[1]]
    a, an, cb, ce = own[0]
    o = np.argsort(key, kind='stable')
    cnt = np.bincount(g.et[o][cb:ce], minlength=g.R2)
    n255 = int((cnt >= 255).sum())
    if saturated:
        assert n255 > K_HOT[bwd], n255
    else:
        assert n_rels == K_HOT[bwd] and int((cnt > 0).sum()) >= n255 == K_HOT[bwd], (n255, int((cnt > 0).sum()))


# ---- device side ------------------------------------------------------------------------------------------------------------
def i32(a, cap=0):
    t = torch.zeros(max(len(a), cap, 1), dtype=torch.int32)
    t[:len(a)] = torch.from_numpy(np.asarray(a, dtype=np.int32))
    return t.to(DEV)


def fwd_structs(g, cap=0):
    return i32(g.rp_dst), i32(g.src, cap), i32(g.et, cap)


def bwd_structs(g):
    o = np.argsort(g.src, kind='stable')
    r = np.argsort(g.et, kind='stable')
    return (i32(g.rp_src), i32(g.dst[o]), i32(g.et[o]), i32(g.ptr(g.et, g.R2)), i32(g.src[r]), i32(g.dst[r]))


def make_inputs(g, indexed, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    X = torch.randn(ENT_ROWS if indexed else g.n_src, 200, device=DEV, generator=gen) * 0.5
    h_index = None
    if indexed:                                    # half of the rows repeat 64 entities
        h_index = torch.randint(0, ENT_ROWS, (g.n_src,), device=DEV, generator=gen, dtype=torch.int32)
        few = torch.randint(0, 64, (g.n_src,), device=DEV, generator=gen, dtype=torch.int32)
        h_index = torch.where(torch.rand(g.n_src, device=DEV, generator=gen) < 0.5, few, h_index)
    W = torch.randn(g.R2, 400, device=DEV, generator=gen) * 0.3
    if g.norm is not None:
        norm = g.norm
    else:                                          # never 1, so a dropped scale shows on single-edge rows too
        deg = torch.from_numpy(np.maximum(np.bincount(g.dst, minlength=g.n_dst), 1)).to(DEV)
        norm = (0.5 + torch.rand(g.n_dst, device=DEV, generator=gen)) / deg
    return gen, X, h_index, W, norm.float().contiguous()


def sentinel(rows):
    return torch.arange(rows * 200, device=DEV, dtype=torch.float32).view(rows, 200) * 0.5 - 7.0


@contextlib.contextmanager
def deterministic(on=True):
    from renet_b200 import _lib
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        _lib.stream()
        assert _lib.lib().renet_get_deterministic() == int(on)
        yield
    finally:
        torch.use_deterministic_algorithms(before)
        _lib.stream()


def kernels_of(fn):
    """{(kernel, template booleans)} of the library's rgcn_* kernels that fn launches"""
    # a trace that lost its records (no rgcn kernel at all) is taken again; in a process that has run many traces the
    # records lost are those at the edges of a trace, so fn runs between two torch kernels (their names are not matched)
    prime = torch.zeros(1, device=DEV)
    for _ in range(10):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            prime.add_(1)
            torch.cuda.synchronize()
            fn()
            torch.cuda.synchronize()
            prime.add_(1)
            torch.cuda.synchronize()
        events = [ev for ev in prof.events() if 'kernel' in ev.name and re.search(r'rgcn_\w+_kernel', ev.name)]
        if events:
            break
    seen = set()
    for ev in events:
        m = re.search(r'rgcn_\w+_kernel', ev.name)
        if m:
            flags = re.findall(r'true|false|\(bool\)[01]', ev.name[m.end():].split('(float', 1)[0].split('(const', 1)[0])
            n = {'rgcn_gather_stream_kernel': 4, 'rgcn_gather_d200_kernel': 3, 'rgcn_dh_tile_kernel': 2,
                 'rgcn_dw_d200_kernel': 2}.get(m.group(0), 0)
            assert len(flags) >= n, ev.name
            seen.add((m.group(0), tuple(f in ('true', '(bool)1') for f in flags[:n])))
    return seen


def assert_kernels(case, fn, expected):
    seen = kernels_of(fn)
    assert seen == expected, '%s: ran %s, expected %s' % (case, sorted(seen), sorted(expected))


def fwd_kernel(which, relu, loop, indexed):
    if which == 'stream':
        return {('rgcn_gather_stream_kernel', (relu, loop, indexed, False))}
    return {('rgcn_gather_d200_kernel', (relu, loop, indexed))}


def bwd_kernels(which, loop, indexed, det):
    dh = ('rgcn_gather_stream_kernel', (False, loop, False, True)) if which == 'stream' else ('rgcn_dh_tile_kernel', (loop, det))
    return {dh, ('rgcn_dw_d200_kernel', (indexed, det))} | ({('rgcn_dw_reduce_kernel', ())} if det else set())


# ---- float64 reference -------------------------------------------------------------------------------------------------------
CHUNK = 16384


def _edges(g):
    """g's src, dst, type as int64 device tensors (g may hold numpy arrays or device tensors)"""
    return (torch.as_tensor(a, device=DEV).long() for a in (g.src, g.dst, g.et))


def ref_forward(g, X, h_index, W, norm, loop, chunk=CHUNK):
    """(pre-activation reference, S) [n_dst, 200] in float64; chunk: edges per pass (a pass holds ~ 1.6 KB of float64
    messages per edge)"""
    src, dst, et = _edges(g)
    rows = h_index.long()[src] if h_index is not None else src
    acc = torch.zeros(2, g.n_dst, 100, 2, dtype=torch.float64, device=DEV)
    for a in range(0, g.E, chunk):                 # block b / in i / out j at b*4 + i*2 + j
        b = slice(a, a + chunk)
        x, w = X[rows[b]].double().view(-1, 100, 2), W[et[b]].double().view(-1, 100, 2, 2)
        acc[0].index_add_(0, dst[b], torch.einsum('ebi,ebij->ebj', x, w))
        acc[1].index_add_(0, dst[b], torch.einsum('ebi,ebij->ebj', x.abs(), w.abs()))
    acc = acc.view(2, g.n_dst, 200) * norm.double()[None, :, None]
    if g.E == 0:                                   # DGL's pass-through: the reduce is skipped, h stays
        h = X[h_index.long()] if h_index is not None else X
        acc[0] = h.double() * norm.double()[:, None]
        acc[1] = acc[0].abs()
    if loop is not None:
        return acc[0] + loop.double(), acc[1].abs() + loop.double().abs()
    return acc[0], acc[1].abs()


def ref_backward(g, X, h_index, W, norm, P, chunk=CHUNK):
    """(dH, S_dH [n_src, 200], dW, S_dW [R2, 400]) in float64, without the self-loop part and the base"""
    src, dst, et = _edges(g)
    rows = h_index.long()[src] if h_index is not None else src
    G = P.double() * norm.double()[:, None]
    dH = torch.zeros(2, g.n_src, 100, 2, dtype=torch.float64, device=DEV)
    dW = torch.zeros(2, g.R2, 400, dtype=torch.float64, device=DEV)
    for a in range(0, g.E, chunk):
        b = slice(a, a + chunk)
        x, w = X[rows[b]].double().view(-1, 100, 2), W[et[b]].double().view(-1, 100, 2, 2)
        gg = G[dst[b]].view(-1, 100, 2)
        dH[0].index_add_(0, src[b], torch.einsum('ebij,ebj->ebi', w, gg))
        dH[1].index_add_(0, src[b], torch.einsum('ebij,ebj->ebi', w.abs(), gg.abs()))
        dW[0].index_add_(0, et[b], torch.einsum('ebi,ebj->ebij', x, gg).reshape(-1, 400))
        dW[1].index_add_(0, et[b], torch.einsum('ebi,ebj->ebij', x.abs(), gg.abs()).reshape(-1, 400))
    dH = dH.view(2, g.n_src, 200)
    return dH[0], dH[1], dW[0], dW[1]


def bar_ratio(got, ref, S, n):
    """(per row: the largest err / ((n + 4) 2^-24 S) over the row's elements, |got - ref|); n: int64 device tensor"""
    unit = U * (n.double() + 4)[:, None] * S
    err = (got.double() - ref).abs()
    ratio = torch.where(unit > 0, err / unit.clamp_min(1e-300), torch.where(err > 0, float('inf'), 0.0).double())
    return ratio.max(1).values, err


def check_rows(label, case, what, got, ref, S, n_terms, exact_to=None):
    """per-row bar; rows with n_terms == 0 must equal exact_to bit for bit"""
    n = torch.as_tensor(n_terms, device=DEV).long() if torch.is_tensor(n_terms) else torch.from_numpy(
        np.asarray(n_terms, dtype=np.int64)).to(DEV)
    assert torch.isfinite(got).all(), (case, what, 'not finite')
    if exact_to is not None:
        z = (n == 0).nonzero().flatten()
        bad = (got[z] != exact_to[z]).any(1).nonzero().flatten()
        assert bad.numel() == 0, '%s %s: row %d has no edges and is not bit-equal to its self-loop row / base' % (
            case, what, int(z[bad[0]]))
    per_row, err = bar_ratio(got, ref, S, n)
    worst = float(per_row.max())
    row = int(per_row.argmax())
    if worst > WORST.get(label, (-1.0,))[0]:
        WORST[label] = (worst, case, what, row, int(n[row]))
    assert worst <= C, '%s %s (%s): row %d with n = %d is %.3g x (n + 4) 2^-24 S off (|err| %.3g); %d rows fail' % (
        case, what, label, row, int(n[row]), worst, float(err[row].max()), int((per_row > C).sum()))


# ---- forward ----------------------------------------------------------------------------------------------------------------
def run_fwd(case, g, expect, relu, loop, indexed, api='gather', hots=(), e_launch=None, seed=1):
    """api 'gather': renet_rgcn_gather[_hot] with random self-loop rows in the output; 'block': renet_rgcn_block_fwd, the
    self-loop rows from renet_selfloop_gemm on the same operands.  hots: relation lists for renet_rgcn_gather_hot, each
    result torch.equal to the list-free one."""
    from renet_b200 import _lib
    L, P = _lib.lib(), _lib.ptr
    N, E = g.n_dst, g.E
    e_launch = E if e_launch is None else e_launch
    gen, X, h_index, W, norm = make_inputs(g, indexed, seed)
    rp, cs, ct = fwd_structs(g, e_launch)
    Wloop = looprows = None
    if loop and api == 'block':
        Wloop = torch.randn(200, 200, device=DEV, generator=gen) * 0.07
        looprows = torch.empty(N, 200, device=DEV)
        _lib.check(L.renet_selfloop_gemm(P(X), P(h_index), P(Wloop), P(looprows), N, 200, 200, _lib.stream()), 'selfloop')
    elif loop:
        looprows = torch.randn(N, 200, device=DEV, generator=gen) * 0.3
    assert api == 'gather' or loop
    tail = sentinel(EXTRA)

    def call(hot=None):
        out = torch.full((N + EXTRA, 200), float('nan'), device=DEV)
        out[N:] = tail
        if api == 'block':
            rc = L.renet_rgcn_block_fwd(P(X), P(h_index), P(W), P(Wloop), P(rp), P(cs), P(ct), P(norm), P(out), N, e_launch, 200,
                                        200, 100, g.R2, int(relu), _lib.stream())
        else:
            if loop:
                out[:N] = looprows
            if hot is None:
                rc = L.renet_rgcn_gather(P(X), P(h_index), P(W), P(rp), P(cs), P(ct), P(norm), P(out), N, e_launch, 200, 200, 100,
                                         g.R2, int(relu), int(loop), _lib.stream())
            else:
                h, n = hot
                rc = L.renet_rgcn_gather_hot(P(X), P(h_index), P(W), P(rp), P(cs), P(ct), P(norm), P(out), N, e_launch, 200, 200,
                                             100, g.R2, int(relu), int(loop), P(h), n, _lib.stream())
        _lib.check(rc, 'forward')
        return out

    got = call()
    assert_kernels(case, call, fwd_kernel(expect, relu, loop, indexed))
    for ids in hots:
        hot = (i32(ids), len(ids))
        assert torch.equal(call(hot), got), (case, 'hot list', list(ids)[:8])
    if hots:
        assert_kernels(case, lambda: call((i32(hots[-1]), len(hots[-1]))), fwd_kernel(expect, relu, loop, indexed))
    assert torch.equal(got[N:], tail), (case, 'rows past N were written')
    got = got[:N]
    ref, S = ref_forward(g, X, h_index, W, norm, looprows)
    act = (lambda t: t.clamp_min(0)) if relu else (lambda t: t)
    exact = act(looprows) if loop else torch.zeros(N, 200, device=DEV)
    n_terms = np.diff(g.rp_dst) if E else np.ones(N, dtype=np.int64)
    check_rows(expect + ' forward', case, 'Hout', got, act(ref), S, n_terms, exact)
    return got


# ---- backward ---------------------------------------------------------------------------------------------------------------
def run_bwd(case, g, expect, relu, loop, indexed, det=False, bipartite=False, seed=2):
    from renet_b200 import _lib
    L, P = _lib.lib(), _lib.ptr
    Ns, Nd, E, R2 = g.n_src, g.n_dst, g.E, g.R2
    assert E > 0 and (bipartite or Ns == Nd) and not (bipartite and (loop or indexed))
    gen, X, h_index, W, norm = make_inputs(g, indexed, seed)
    Wloop = torch.randn(200, 200, device=DEV, generator=gen) * 0.07 if loop else None
    dout = torch.randn(Nd, 200, device=DEV, generator=gen)
    Hout = None
    if relu:                                       # the kernel's own forward output decides the mask
        rp, cs, ct = fwd_structs(g)
        Hout = torch.empty(Nd, 200, device=DEV)
        if bipartite:
            rc = L.renet_rgcn_gather(P(X), None, P(W), P(rp), P(cs), P(ct), P(norm), P(Hout), Nd, E, 200, 200, 100, R2, 1, 0,
                                     _lib.stream())
        else:
            rc = L.renet_rgcn_block_fwd(P(X), P(h_index), P(W), P(Wloop), P(rp), P(cs), P(ct), P(norm), P(Hout), Nd, E, 200, 200,
                                        100, R2, 1, _lib.stream())
        _lib.check(rc, 'forward for the mask')
    Pm = dout * (Hout > 0) if relu else dout
    t_rp, t_cd, t_ct, r_rp, r_src, r_dst = bwd_structs(g)
    base_W = torch.randn(R2, 400, device=DEV, generator=gen) * 1e-2
    base_Wl = torch.randn(200, 200, device=DEV, generator=gen) * 1e-2 if loop else None
    ws = torch.empty(((Nd * 200 + 3) // 4) * 4 + 200 * 200, device=DEV)
    tail = sentinel(EXTRA)

    def call():
        dH = torch.full((Ns + EXTRA, 200), float('nan'), device=DEV)
        dH[Ns:] = tail
        dW, dWl = base_W.clone(), (base_Wl.clone() if loop else None)
        if bipartite:
            rc = L.renet_rgcn_bipartite_bwd(P(X), P(W), P(t_rp), P(t_cd), P(t_ct), P(r_rp), P(r_src), P(r_dst), P(norm), P(Hout),
                                            P(dout), P(dH), P(dW), P(ws), Ns, Nd, E, 200, 200, 100, R2, int(relu), _lib.stream())
        else:
            rc = L.renet_rgcn_block_bwd(P(X), P(h_index), P(W), P(Wloop), P(t_rp), P(t_cd), P(t_ct), P(r_rp), P(r_src), P(r_dst),
                                        P(norm), P(Hout), P(dout), P(dH), P(dW), P(dWl), P(ws), Ns, E, 200, 200, 100, R2,
                                        int(relu), _lib.stream())
        _lib.check(rc, 'backward')
        return dH, dW, dWl

    dH_loop = torch.zeros(Ns, 200, device=DEV)
    with deterministic(det):
        dH, dW, dWl = call()
        if det:
            again = call()
            assert all(torch.equal(a, b) for a, b in zip((dH, dW), again)), (case, 'deterministic mode: two runs differ')
            assert not loop or torch.equal(dWl, again[2])
        assert_kernels(case, call, bwd_kernels(expect, loop, indexed, det))
        if loop:                                   # the dense self-loop part of dH, from the GEMM engine on the same operands
            scratch = torch.zeros(200, 200, device=DEV)
            _lib.check(L.renet_selfloop_gemm_bwd(P(X), P(h_index), P(Wloop), P(Pm), P(dH_loop), P(scratch), P(ws[-40000:]), Ns, 200,
                                                 200, _lib.stream()), 'selfloop bwd')
    assert torch.equal(dH[Ns:], tail), (case, 'rows of dH past N were written')
    dH = dH[:Ns]
    rH, sH, rW, sW = ref_backward(g, X, h_index, W, norm, Pm)
    label = ('stream dH' if expect == 'stream' else 'tile dH') + (' det' if det and expect == 'tile' else '')
    check_rows(label, case, 'dH', dH, rH + dH_loop.double(), sH + dH_loop.double().abs(), np.diff(g.rp_src), dH_loop)
    check_rows('dW det' if det else 'dW', case, 'dW', dW, rW + base_W.double(), sW + base_W.double().abs(),
               np.bincount(g.et, minlength=R2), base_W)
    if loop:
        Xr = X[h_index.long()] if indexed else X
        refl = Xr.double().t() @ Pm.double()
        assert float(((dWl.double() - base_Wl.double()) - refl).abs().max()) <= 2e-5 * float(refl.abs().max()), (case, 'dWloop')


# ---- the cases ---------------------------------------------------------------------------------------------------------------
CASES = {}


def case(name):
    def reg(fn):
        assert name not in CASES
        CASES[name] = functools.partial(fn, name)
        return fn
    return reg


def both(name, build, expect, fwd=None, bwd=None):
    """a forward case on build('dst') and a backward one on the same degree sequence as out-degrees, build('src')"""
    fwd, bwd = fwd or {}, bwd or {}

    @case(name + '-fwd')
    def _f(cs):
        run_fwd(cs, build('dst'), expect, **{'relu': True, 'loop': True, 'indexed': False, **fwd})

    @case(name + '-bwd')
    def _b(cs):
        run_bwd(cs, build('src'), expect, **{'relu': True, 'loop': False, 'indexed': False, **bwd})


# stream kernel: row_ptr from global memory
def _rp_global(by):
    N = 40000
    deg = np.zeros(N, dtype=np.int64)
    deg[:N // 2] = exact_degrees(N // 2, 260000, 3)
    deg[N // 2::8] = 1
    g = graph_by_degrees(deg, N, 460, 4, 'zipf', by)
    assert_rp_from_global(g.rp_dst if by == 'dst' else g.rp_src)
    return g


both('rp-global', _rp_global, 'stream', bwd={'loop': True})


@case('rp-global-fwd-indexed')
def _(cs):
    run_fwd(cs, _rp_global('dst'), 'stream', relu=False, loop=False, indexed=True)


# stream kernel: a row heavier than a CTA's share
def _hub(where, by):
    deg = mid_degrees().copy()
    N = len(deg)
    hub = {'mid': N // 2, 'first': 7, 'last': N - 10}[where]
    if where == 'first':
        deg[7] = 6000
    elif where == 'last':
        deg[N - 10] = 6000
    else:
        deg[hub] = 6000
    g = graph_by_degrees(deg, N, 460, 5, 'zipf', by)
    assert_hub(g.rp_dst if by == 'dst' else g.rp_src, hub, where == 'first', where == 'last')
    return g


for _w in ('mid', 'first', 'last'):
    both('hub-' + _w, functools.partial(_hub, _w), 'stream', bwd={'loop': _w == 'mid'})


# stream kernel: relation-id range against the resident-row table
def _r2(R2, how, by):
    return graph_by_degrees(mid_degrees(), 20000, R2, 6, how, by)


for _R2f, _R2b, _how in ((1, 1, 'uniform'), (40, 40, 'uniform'), (82, 77, 'uniform'), (83, 78, 'uniform'), (83, 78, 'zipf'),
                         (512, 512, 'uniform'), (512, 512, 'zipf'), (2048, 2048, 'uniform'), (2049, 2049, 'uniform'),
                         (2049, 2049, 'zipf')):
    @case('r2-%d-%s-fwd' % (_R2f, _how))
    def _(cs, R2=_R2f, how=_how):
        run_fwd(cs, _r2(R2, how, 'dst'), 'stream', relu=True, loop=True, indexed=False)

    @case('r2-%d-%s-bwd' % (_R2b, _how))
    def _(cs, R2=_R2b, how=_how):
        run_bwd(cs, _r2(R2, how, 'src'), 'stream', relu=False, loop=False, indexed=False)


def _hist(saturated, by):
    bwd = by == 'src'
    deg = mid_degrees().copy()
    hub = 9000
    deg[hub] = 25000
    n_rels = 90 if saturated else K_HOT[bwd]
    g = graph_by_degrees(deg, 20000, 460, 7, 'uniform', by, hub=hub, hub_rels=n_rels)
    assert_histogram(g, bwd, hub, n_rels, saturated)
    return g


both('hist-saturated', functools.partial(_hist, True), 'stream')
both('hist-exact', functools.partial(_hist, False), 'stream')


@case('hot-lists')
def _(cs):
    g = graph_by_degrees(mid_degrees(), 20000, 460, 8, 'zipf', 'dst')
    freq = np.argsort(-np.bincount(g.et, minlength=460))
    lists = [freq[:1], freq[:82], freq[:83], freq[:200], np.concatenate(([-1, 460], freq[:40], [460, -1, -7, 1 << 20])),
             np.asarray([7, 7, 7, 3, 3] * 10), freq[::-1][:82]]
    assert [len(x) for x in lists[:4]] == [1, 82, 83, 200]
    got = run_fwd(cs, g, 'stream', relu=True, loop=True, indexed=False, hots=lists)
    # a list of length 0 behind a non-null pointer is "no list"
    from renet_b200 import _lib
    L, P = _lib.lib(), _lib.ptr
    gen, X, h_index, W, norm = make_inputs(g, False, 1)
    rp, ccs, ct = fwd_structs(g)
    out = torch.randn(g.n_dst, 200, device=DEV, generator=gen) * 0.3
    _lib.check(L.renet_rgcn_gather_hot(P(X), None, P(W), P(rp), P(ccs), P(ct), P(norm), P(out), g.n_dst, g.E, 200, 200, 100, 460, 1,
                                       1, P(i32([5])), 0, _lib.stream()), 'gather_hot')
    assert torch.equal(out, got)


# every instantiation
for _r in (0, 1):
    for _l in (0, 1):
        for _i in (0, 1):
            @case('inst-stream-fwd-%d%d%d' % (_r, _l, _i))
            def _(cs, r=_r, l=_l, i=_i):
                run_fwd(cs, graph_by_degrees(mid_degrees(), 20000, 460, 9, 'zipf'), 'stream', relu=bool(r), loop=bool(l),
                        indexed=bool(i), api='block' if l else 'gather')

            @case('inst-tile-fwd-%d%d%d' % (_r, _l, _i))
            def _(cs, r=_r, l=_l, i=_i):
                run_fwd(cs, graph_by_degrees(mid_degrees(1500), 1500, 460, 10, 'zipf'), 'tile', relu=bool(r), loop=bool(l),
                        indexed=bool(i), api='block' if l and r else 'gather')
for _l in (0, 1):
    @case('inst-stream-bwd-loop%d' % _l)
    def _(cs, l=_l):
        run_bwd(cs, graph_by_degrees(mid_degrees(), 20000, 460, 11, 'zipf', 'src'), 'stream', relu=True, loop=bool(l),
                indexed=True)
    for _d in (0, 1):
        @case('inst-tile-bwd-loop%d%s' % (_l, '-det' if _d else ''))
        def _(cs, l=_l, d=_d):
            run_bwd(cs, graph_by_degrees(mid_degrees(1500), 1500, 460, 12, 'zipf', 'src'), 'tile', relu=True, loop=bool(l),
                    indexed=bool(l), det=bool(d))


# selection boundaries
def _edge(N, E, by):
    return graph_by_degrees(exact_degrees(N, E, N + E), N, 460, 13, 'zipf', by)


for _N, _idx, _exp in ((2047, False, 'tile'), (2048, False, 'stream'), (16383, True, 'tile'), (16384, True, 'stream'),
                       (40960, False, 'stream'), (40961, False, 'tile'), (40960, True, 'stream'), (40961, True, 'tile')):
    @case('edge-n%d-%s-fwd' % (_N, 'indexed' if _idx else 'plain'))
    def _(cs, N=_N, idx=_idx, exp=_exp):
        run_fwd(cs, _edge(N, 60000, 'dst'), exp, relu=True, loop=True, indexed=idx)
for _N, _exp in ((16383, 'tile'), (16384, 'stream'), (40960, 'stream'), (40961, 'tile')):
    @case('edge-n%d-bwd' % _N)
    def _(cs, N=_N, exp=_exp):
        run_bwd(cs, _edge(N, 60000, 'src'), exp, relu=True, loop=False, indexed=False)
for _E, _exp in ((16383, 'tile'), (16384, 'stream')):
    @case('edge-e%d-fwd' % _E)
    def _(cs, E=_E, exp=_exp):
        run_fwd(cs, _edge(20000, E, 'dst'), exp, relu=True, loop=True, indexed=True)

    @case('edge-e%d-bwd' % _E)
    def _(cs, E=_E, exp=_exp):
        run_bwd(cs, _edge(20000, E, 'src'), exp, relu=True, loop=False, indexed=False)


@case('edge-capacity-fwd')
def _(cs):
    g = _edge(20000, 5000, 'dst')
    run_fwd(cs, g, 'tile', relu=False, loop=True, indexed=False)
    run_fwd(cs, g, 'stream', relu=False, loop=True, indexed=False, e_launch=4 * g.E)


# layer 2 at production shape
@functools.lru_cache(maxsize=1)
def _readout():
    from renet_b200.graph import ReadoutSubgraph

    class Parent:
        pass
    N, S = 34000, 8000
    rng = np.random.default_rng(14)
    deg = rng.integers(0, 25, N)
    p = Parent()
    p.device, p.N = torch.device(DEV), N
    rp = np.concatenate(([0], np.cumsum(deg)))
    E = int(rp[-1])
    p.row_ptr, p.col_src = i32(rp), i32(rng.integers(0, N, E))
    ct = i32((rng.zipf(1.3, E) - 1) % 460)
    p.col_type = lambda reverse: ct
    p.norm = torch.from_numpy((1.0 / np.maximum(deg, 1)).astype(np.float32)).to(DEV)
    nodes = rng.choice(N, 7000, replace=False)
    sub = ReadoutSubgraph(p, i32(np.concatenate((nodes, rng.choice(nodes, S - 7000)))), False)
    n_uniq, E2 = sub.sizes()
    srp = sub.row_ptr.cpu().numpy().astype(np.int64)
    assert n_uniq == 7000 and sub.N == S and int(srp[-1]) == E2 and 70000 < E2 < 110000
    dst = np.repeat(np.arange(S), np.diff(srp))
    g = Graph(N, S, 460, sub.col_src[:E2].cpu().numpy(), dst, sub.col_type(False)[:E2].cpu().numpy(), norm=sub.norm.clone())
    assert np.array_equal(g.rp_dst, srp)
    return g, sub.E_cap


@case('readout-fwd')
def _(cs):
    g, cap = _readout()
    run_fwd(cs, g, 'stream', relu=False, loop=True, indexed=False, e_launch=cap)


for _d in (0, 1):
    @case('readout-bwd' + ('-det' if _d else ''))
    def _(cs, d=_d):
        run_bwd(cs, _readout()[0], 'stream', relu=False, loop=False, indexed=False, det=bool(d), bipartite=True)


# tile kernels
def _tile_deg(kind):
    rng = np.random.default_rng(15)
    if kind.startswith('n'):
        deg = rng.integers(0, 7, int(kind[1:]))
        deg[0] = max(deg[0], 3)
    elif kind == 'span8':
        deg = np.zeros(16, dtype=np.int64)
        deg[:3] = [2, 400, 3]
        chunk = -(-405 // 8)                        # the warps' slices: all 8 hold edges of row 1 (edges 2 .. 401)
        assert all(max(w * chunk, 2) < min((w + 1) * chunk, 402) for w in range(8))
    else:                                          # 'hole'
        deg = np.concatenate((rng.integers(3, 9, 16), np.zeros(16, dtype=np.int64), rng.integers(3, 9, 16)))
    return deg


for _k in ('n1', 'n15', 'n16', 'n17', 'n33', 'span8', 'hole'):
    @case('tile-%s-fwd' % _k)
    def _(cs, k=_k):
        deg = _tile_deg(k)
        g = graph_by_degrees(deg, len(deg), 460, 16)
        run_fwd(cs, g, 'tile', relu=True, loop=True, indexed=False, api='block')
        run_fwd(cs, g, 'tile', relu=False, loop=False, indexed=True)
    for _d in (0, 1):
        @case('tile-%s-bwd%s' % (_k, '-det' if _d else ''))
        def _(cs, k=_k, d=_d):
            deg = _tile_deg(k)
            g = graph_by_degrees(deg, len(deg), 460, 17, by='src')
            run_bwd(cs, g, 'tile', relu=True, loop=True, indexed=False, det=bool(d))
            run_bwd(cs, g, 'tile', relu=False, loop=False, indexed=True, det=bool(d))
for _i in (0, 1):
    @case('tile-e0-' + ('indexed' if _i else 'plain'))
    def _(cs, i=_i):
        g = graph_by_degrees(np.zeros(33, dtype=np.int64), 33, 460, 18)
        run_fwd(cs, g, 'tile', relu=True, loop=True, indexed=bool(i))
        run_fwd(cs, g, 'tile', relu=False, loop=False, indexed=bool(i))


# dW: runs of 64 edges against relation boundaries
DW_COUNTS = {
    'empties': [0, 0, 0, 70, 0, 0, 0, 0, 5, 0, 130, 1, 0, 0, 40, 0, 0],
    'run-edges': [64, 64, 63, 1, 65, 63, 128, 1, 63, 64, 129, 127, 1],     # boundaries at 64, 128, 191, 192, 257, 320, 448, 449, ...
    'singles-hub': [1, 2400, 1, 1, 700, 1, 895, 1],
    '64-singles': [50, 14] + [1] * 64 + [64] + [1] * 64 + [30],
    'e1': [0, 1, 0], 'e63': [0, 63, 0], 'e64': [0, 64, 0], 'e65': [0, 65, 0],
    'r2-1': [200],
}
_c = np.cumsum(DW_COUNTS['run-edges'])
assert {64, 128, 192, 320, 448, 512, 576}.issubset(set(_c)) and {191, 257, 449}.issubset(set(_c))
assert sum(DW_COUNTS['singles-hub']) == 4000 and DW_COUNTS['64-singles'][:2] == [50, 14]
for _k, _counts in DW_COUNTS.items():
    for _d in (0, 1):
        @case('dw-%s%s' % (_k, '-det' if _d else ''))
        def _(cs, counts=_counts, d=_d):
            g = graph_by_relations(counts, 300, 19)
            run_bwd(cs, g, 'tile', relu=True, loop=False, indexed=False, det=bool(d))
            run_bwd(cs, g, 'tile', relu=False, loop=True, indexed=True, det=bool(d))


def summary():
    return ['%-15s worst ratio %.3f  (%s %s, row %d, n = %d)' % ((k,) + WORST[k]) for k in sorted(WORST)]
