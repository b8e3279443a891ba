"""-m "not gpu": the work partition and hand-over protocol of the persistent gather kernel (renet_b200/csrc/rgcn_stream.cuh),
restated in Python line by line and checked for its invariants on many random CSR structures -- the host-checkable half of a
kernel whose arithmetic the -m gpu tests pin:

  * every edge is accumulated by exactly one warp, every destination with in-edges is finished (epilogue) exactly once,
    destinations without in-edges are never touched by the edge pass (a separate all-warps pass writes them);
  * a destination cut by warp boundaries is finished by the warp that started it, after the heads of the following warps
    in warp order, i.e. its edges are summed in CSR order: the result does not depend on scheduling;
  * CTA ranges are node-aligned, contiguous and cover [0, N); warp ranges are contiguous and cover the CTA's edges;
  * the cost model (edges + kStNodeCost per destination) bounds the imbalance between CTAs by the heaviest destination.

The constants mirror the kernel (kStNodeCost = 2, 132 CTAs, 32 warps); if the kernel's partition changes, this file changes
with it."""
import numpy as np
import pytest

NODE_COST, GRID, WARPS = 2, 132, 32


def cta_boundary(rp, N, E, c_idx, grid=GRID):
    """lower_bound of the cost key by rounds of 256 probes, then the nearer of the two destination starts around the
    target (rgcn_stream.cuh: "CTA partition").  Returns (first destination, its row_ptr)."""
    if c_idx <= 0:
        return 0, 0
    if c_idx >= grid:
        return N, E
    total = E + NODE_COST * N
    target = c_idx * total // grid
    lo, hi = 0, N
    rounds = 1 if N < 256 else (2 if N < 65536 else (3 if N < (1 << 24) else 4))
    prev = None
    for r in range(rounds):
        step = (hi - lo) // 256 + 1
        probes = [min(lo + (ht + 1) * step - 1, hi) for ht in range(256)]
        below = [int(rp[p]) + NODE_COST * p < target for p in probes]
        f = sum(below)                                     # keys ascend: the probes below the target are a prefix
        assert below == [True] * f + [False] * (256 - f)
        if r == rounds - 1:
            assert step == 1
            ans, val = lo + f, int(rp[probes[f]])
            assert probes[f] == ans
            prev = int(rp[probes[f - 1]]) if f >= 1 else None
        new_hi = min(lo + (f + 1) * step - 1, hi)
        new_lo = lo if f == 0 else min(lo + f * step - 1, hi) + 1
        lo, hi = new_lo, new_hi
    assert lo == hi == ans
    A, cb = ans, val
    if prev is not None:
        k_hi, k_lo = cb + NODE_COST * A, prev + NODE_COST * (A - 1)
        if k_hi - target > target - k_lo:
            A, cb = A - 1, prev
    return A, cb


def warp_ranges(rp, A, A_next, cb, ce, warps=WARPS):
    """rgcn_stream.cuh "warp ranges": equal shares of (edges + NODE_COST per destination), cut at edge positions."""
    cta_cost = (ce - cb) + NODE_COST * (A_next - A)

    def start(j):
        T = cta_cost * j // warps
        l, h = A, A_next
        while l < h:
            mid = (l + h + 1) >> 1
            if (int(rp[mid]) - cb) + NODE_COST * (mid - A) <= T:
                l = mid
            else:
                h = mid - 1
        if l >= A_next:
            return ce
        r = T - ((int(rp[l]) - cb) + NODE_COST * (l - A))
        return int(rp[l]) + min(r, int(rp[l + 1]) - int(rp[l]))
    e0 = [start(j) for j in range(warps)] + [ce]
    return e0


def run_warp(rp, A, A_next, ce, s_e0, w, log):
    """One warp's pass over its edge range (the loop, `advance`, the end-of-range cases).  log[v] gets ('start', w, edges),
    ('head', w, edges) or ('finish', w) records in program order."""
    e0, e1 = s_e0[w], s_e0[w + 1]
    n = e1 - e0
    # first destination of the range
    l, h = A, A_next
    while h > l:
        mid = (l + h) >> 1
        if int(rp[mid]) >= e0:
            h = mid
        else:
            l = mid + 1
    va = l
    cur, continued = va, False
    if n > 0 and int(rp[va]) > e0:
        cur, continued = va - 1, True
    cur_end = int(rp[cur + 1]) if cur < A_next else ce
    cur_beg = int(rp[cur]) if cur < A_next else ce
    acc = []

    def advance():
        nonlocal cur, cur_beg, cur_end, continued, acc
        if continued:
            log.setdefault(cur, []).append(('head', w, acc))
            continued = False
        elif cur_end > cur_beg:
            log.setdefault(cur, []).append(('start', w, acc))
            log[cur].append(('finish', w))
        else:
            assert not acc                                  # a destination without in-edges: nothing accumulated, nothing written
        acc = []
        cur += 1
        cur_beg = cur_end
        cur_end = int(rp[cur + 1]) if cur < A_next else ce

    for i in range(n):
        while e0 + i >= cur_end:
            advance()
        assert cur_beg <= e0 + i < cur_end or continued
        acc.append(e0 + i)
    if n > 0:
        if cur_end <= e1:
            advance()
        elif continued:
            log.setdefault(cur, []).append(('head', w, acc))
        else:
            # starter of a destination that later warps continue: their heads, in warp order, then the epilogue
            got = list(acc)
            k = w + 1
            waited = []
            while k < WARPS and s_e0[k] < cur_end:
                if s_e0[k + 1] != s_e0[k]:
                    waited.append(k)
                k += 1
            log.setdefault(cur, []).append(('start', w, got))
            log[cur].append(('collect', w, waited))
            log[cur].append(('finish', w))


def check_graph(rp, grid=GRID):
    rp = np.asarray(rp, dtype=np.int64)
    N, E = len(rp) - 1, int(rp[-1])
    bounds = [cta_boundary(rp, N, E, c, grid) for c in range(grid + 1)]
    As = [b[0] for b in bounds]
    assert As[0] == 0 and As[-1] == N and all(a <= b for a, b in zip(As, As[1:]))           # contiguous, node-aligned cover
    for (A, cb) in bounds:
        assert cb == int(rp[A])
    log = {}
    cta_edges = []
    for c in range(grid):
        (A, cb), (A_next, ce) = bounds[c], bounds[c + 1]
        cta_edges.append(ce - cb)
        s_e0 = warp_ranges(rp, A, A_next, cb, ce)
        assert s_e0[0] == cb and s_e0[-1] == ce and all(a <= b for a, b in zip(s_e0, s_e0[1:]))
        for w in range(WARPS):
            run_warp(rp, A, A_next, ce, s_e0, w, log)
    deg = np.diff(rp)
    for v in range(N):
        recs = log.get(v, [])
        if deg[v] == 0:
            assert not recs, v                              # the edge pass never touches destinations without in-edges
            continue
        starts = [r for r in recs if r[0] == 'start']
        heads = sorted((r for r in recs if r[0] == 'head'), key=lambda r: r[1])
        fins = [r for r in recs if r[0] == 'finish']
        assert len(starts) == 1 and len(fins) == 1 and fins[0][1] == starts[0][1], v
        order = list(starts[0][2])
        for h in heads:
            assert h[1] > starts[0][1]
            order += h[2]
        assert order == list(range(int(rp[v]), int(rp[v + 1]))), v          # every edge once, in CSR order
        col = [r for r in recs if r[0] == 'collect']
        if heads:
            assert len(col) == 1 and col[0][2] == [h[1] for h in heads], v  # the starter waits for exactly the warps that publish
        else:
            assert not col or col[0][2] == []
    return np.asarray(cta_edges), deg


def _rand_csr(rng, N, E, kind):
    if kind == 'uniform':
        dst = rng.randint(0, N, E)
    elif kind == 'zipf':
        dst = rng.zipf(1.3, E) % N
    elif kind == 'heavy':
        dst = rng.randint(0, N, E)
        dst[:E // 3] = N // 2                               # one destination with a third of all edges
    else:                                                   # 'sparse': most destinations have no in-edges, also at both ends
        alive = np.sort(rng.choice(np.arange(5, max(6, N - 7)), size=max(1, N // 10), replace=False))
        dst = alive[rng.randint(0, len(alive), E)]
    return np.concatenate(([0], np.cumsum(np.bincount(dst, minlength=N))))


@pytest.mark.parametrize('kind', ['uniform', 'zipf', 'heavy', 'sparse'])
@pytest.mark.parametrize('N,E', [(40, 3000), (300, 9000), (5000, 20000), (70000, 40000)])
def test_partition_and_hand_over_invariants(kind, N, E):
    rng = np.random.RandomState(N + E + len(kind))
    rp = _rand_csr(rng, N, E, kind)
    cta_edges, deg = check_graph(rp)
    assert cta_edges.sum() == E
    if kind in ('uniform', 'zipf') and E >= 9000:
        # node-aligned boundaries rounded to the nearer destination start: a CTA's work is within one heaviest destination
        # (+ the rounding of the cost targets) of the mean
        nodes_per_cta = np.diff([cta_boundary(rp, N, E, c)[0] for c in range(GRID + 1)])
        cost = cta_edges + NODE_COST * nodes_per_cta
        assert np.abs(cost - cost.mean()).max() <= deg.max() + NODE_COST + 2


def test_degenerate_graphs():
    for rp in ([0, 0, 0, 0], [0, 5], [0, 0, 7, 7, 7], [0] + [3] * 200, list(range(0, 600, 2))):
        check_graph(np.asarray(rp))


def test_many_small_random_graphs():
    rng = np.random.RandomState(12345)
    for _ in range(120):
        N = int(rng.randint(1, 400))
        E = int(rng.randint(0, 4000))
        kind = ['uniform', 'zipf', 'heavy', 'sparse'][rng.randint(0, 4)] if N > 20 else 'uniform'
        rp = _rand_csr(rng, N, E, kind) if E > 0 else np.zeros(N + 1, dtype=np.int64)
        cta_edges, _ = check_graph(rp)
        assert cta_edges.sum() == E
