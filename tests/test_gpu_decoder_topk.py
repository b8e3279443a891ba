"""-m gpu: renet_decoder_topk (decoder.decoder_topk), the per-row top-k with exclusion lists, against an fp64 PyTorch
restatement: per row the k largest p = softmax(x @ W^T + b) over the columns outside the row's list, p descending, ties to
the lower column, -1 / 0 past the admissible columns.

Index sets are exact wherever the k-th and (k+1)-th admissible fp64 values differ by more than 1e-5 relative; values are
within 1e-4 relative of fp64; no listed column is ever returned.  The lists cover the cases the threshold must survive:
lists holding the maximum column of many half tiles (a threshold at the k-th partial maximum would lose answers), lists
longer than the row's partial count (threshold 0), fewer than k admissible columns; and k = 1, k = RENET_TOPK_MAX_K,
planted exact ties, a forced capacity retry, M = 0 and M not a multiple of 64.  Without lists the output is
decoder_group_topk's with R = 1, weight 1 and ORDER_VALUE, bit for bit."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _fixture(M, N, K, seed, zscale=3.0):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=gen)
    w = torch.randn(N, K, generator=gen) * (zscale / K ** 0.5)
    b = torch.randn(N, generator=gen) * 0.5
    return x, w, b


def _units(N):
    """[lo, hi) of every (half column tile) unit the first pass reduces: tiles of 200 columns split at 104."""
    out = []
    for t0 in range(0, N, 200):
        for lo, hi in ((t0, t0 + 104), (t0 + 104, t0 + 200)):
            if lo < N:
                out.append((lo, min(hi, N)))
    return out


def _lists(kind, z64, k, rng):
    """Per-row ascending exclusion lists of the given kind, as python lists."""
    M, N = z64.shape
    out = []
    for m in range(M):
        z = z64[m].cpu().numpy()
        if kind == 'unit_max':           # the maximum column of the k best units: a threshold at rank k would lose answers
            maxima = [lo + int(np.argmax(z[lo:hi])) for lo, hi in _units(N)]
            maxima.sort(key=lambda c: -z[c])
            cols = maxima[:k]
        elif kind == 'long':             # longer than the partial count: threshold 0
            cols = rng.choice(N, size=len(_units(N)) + 7, replace=False)
        elif kind == 'few_left':         # fewer than k admissible columns
            cols = rng.choice(N, size=N - k // 2, replace=False)
        elif kind == 'random':
            cols = rng.choice(N, size=int(rng.randint(0, min(3 * k, N - k) + 1)), replace=False)
        else:
            cols = []
        if m % 7 == 3:
            cols = []                    # some rows without a list
        out.append(sorted(int(c) for c in cols))
    return out


def _device_lists(lists, dup=False):
    """(col, begin, end) int32 on the device; ``dup`` repeats every entry (duplicates only loosen the bound)."""
    col, begin, end = [], [], []
    for cols in lists:
        if dup:
            cols = sorted(cols + cols)
        begin.append(len(col))
        col += cols
        end.append(len(col))
    t = lambda a: torch.tensor(a, dtype=torch.int32, device=DEV)        # noqa: E731
    return t(col if col else [0]), t(begin), t(end)


def _check(vals, idx, z64, lists, k):
    """The fp64 comparison of the module docstring; returns the number of rows in the near-tie band."""
    p64 = torch.softmax(z64, dim=1).cpu()
    vals, idx = vals.cpu(), idx.cpu()
    M, N = p64.shape
    n_band = 0
    for m in range(M):
        banned = set(lists[m]) if lists is not None else set()
        adm = np.array([c for c in range(N) if c not in banned], dtype=np.int64)
        pa = p64[m, adm].numpy()
        order = adm[np.lexsort((adm, -pa))]
        kk = min(k, len(adm))
        got = idx[m].numpy()
        assert (got[kk:] == -1).all() and (vals[m, kk:] == 0).all(), m
        assert (got[:kk] >= 0).all() and not (set(got[:kk].tolist()) & banned), m
        assert len(set(got[:kk].tolist())) == kk
        ref = p64[m, got[:kk]].double()
        assert float(((vals[m, :kk].double() - ref).abs() / ref.clamp_min(1e-300)).max()) <= 1e-4, m
        v = vals[m, :kk]
        assert bool((v[1:] <= v[:-1]).all()), m                               # p descending
        tie = (v[1:] == v[:-1]).numpy()
        assert (got[1:kk][tie] > got[:kk - 1][tie]).all(), m                 # equal values: lower column first
        ps = p64[m, order].numpy()
        if kk < len(adm) and ps[kk - 1] - ps[kk] <= 1e-5 * ps[kk - 1]:
            n_band += 1
            assert p64[m, got[:kk]].min() >= ps[kk - 1] * (1 - 1e-4), m      # still among the near-tie values
        else:
            assert set(got[:kk].tolist()) == set(order[:kk].tolist()), m
    return n_band


CASES = [  # (M, N, K, k, list kind)
    (130, 1000, 64, 10, 'random'),          # M not a multiple of 64
    (64, 23033, 600, 50, 'unit_max'),       # ICEWS18 |E|: the k best units' maxima are all excluded
    (40, 7691, 600, 100, 'unit_max'),       # GDELT |E|
    (48, 1000, 200, 10, 'long'),            # lists longer than the partial count: threshold 0
    (33, 1000, 200, 10, 'few_left'),        # N - L < k: padded rows
    (70, 23033, 600, 1, 'unit_max'),        # k = 1
    (3, 23033, 200, 16384, 'random'),       # k = RENET_TOPK_MAX_K
    (50, 2000, 200, 40, 'none'),
]


@pytest.mark.parametrize('M,N,K,k,kind', CASES)
def test_decoder_topk_vs_fp64(M, N, K, k, kind):
    from renet_b200.decoder import decoder_topk
    x, w, b = (t.to(DEV) for t in _fixture(M, N, K, seed=M + N + K + k))
    z64 = x.double() @ w.double().t() + b.double()
    lists = _lists(kind, z64, k, np.random.RandomState(k))
    ex = _device_lists(lists) if kind != 'none' else None
    runs = [decoder_topk(x, w, b, k, ex) for _ in range(2)]
    vals, idx = runs[0]
    assert vals.shape == (M, k) and idx.shape == (M, k) and idx.dtype == torch.int64 and vals.dtype == torch.float32
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])           # bitwise repeatable
    n_band = _check(vals, idx, z64, lists if ex is not None else None, k)
    assert n_band <= max(1, M // 10), n_band
    if kind == 'few_left':
        assert bool((idx == -1).any(dim=1).sum() >= M // 2)
    if ex is not None:                   # duplicated list entries loosen the threshold only: the same output
        dv, di = decoder_topk(x, w, b, k, _device_lists(lists, dup=True))
        assert torch.equal(dv, vals) and torch.equal(di, idx)


@pytest.mark.parametrize('M,N,K,k', [(130, 1000, 64, 10), (64, 23033, 600, 100), (5, 2000, 200, 1000)])
def test_without_lists_equals_group_topk(M, N, K, k):
    from renet_b200.decoder import ORDER_VALUE, decoder_group_topk, decoder_topk
    x, w, b = (t.to(DEV) for t in _fixture(M, N, K, seed=3))
    ones = torch.ones(M, device=DEV)
    gv, gi = decoder_group_topk(x, w, b, ones, 1, k, ORDER_VALUE)
    v, i = decoder_topk(x, w, b, k)
    assert torch.equal(v, gv) and torch.equal(i, gi)
    empty = _device_lists([[] for _ in range(M)])                # empty lists: the same
    v2, i2 = decoder_topk(x, w, b, k, empty)
    assert torch.equal(v2, gv) and torch.equal(i2, gi)


def test_planted_ties_go_to_the_lower_column():
    """Duplicated W rows and biases give bit-equal logits; the pair straddles the k-th place of many rows."""
    from renet_b200.decoder import decoder_topk
    M, N, K, k = 96, 3000, 200, 20
    x, w, b = _fixture(M, N, K, seed=11)
    rng = np.random.RandomState(5)
    pairs = [(int(a), int(c)) for a, c in zip(rng.choice(1500, 40, replace=False), 1500 + rng.choice(1500, 40, replace=False))]
    for a, c in pairs:
        w[c], b[c] = w[a], b[a]
    x, w, b = x.to(DEV), w.to(DEV), b.to(DEV)
    z64 = x.double() @ w.double().t() + b.double()
    lists = _lists('random', z64, k, rng)
    vals, idx = decoder_topk(x, w, b, k, _device_lists(lists))
    _check(vals, idx, z64, lists, k)
    seen = 0
    for m in range(M):
        got = idx[m].tolist()
        for a, c in pairs:
            if a in lists[m] or c in lists[m]:
                continue
            if c in got:                               # the higher column only after the lower one
                assert a in got and got.index(a) < got.index(c), (m, a, c)
                seen += 1
    assert seen > 0


def test_capacity_retry_gives_the_same_output():
    """A candidate buffer of k is too small (the excluded columns are candidates too): the call reports it and the wrapper
    repeats it with the size reported."""
    from renet_b200 import _lib
    from renet_b200.decoder import decoder_topk
    M, N, K, k = 64, 23033, 600, 50
    x, w, b = (t.to(DEV) for t in _fixture(M, N, K, seed=9))
    z64 = x.double() @ w.double().t() + b.double()
    col, begin, end = _device_lists(_lists('unit_max', z64, k, np.random.RandomState(0)))
    L, P = _lib.lib(), _lib.ptr
    vals = torch.empty(M, k, device=DEV)
    idx = torch.empty(M, k, dtype=torch.int32, device=DEV)
    needed = torch.zeros(1, dtype=torch.int32, device=DEV)
    nbytes = int(L.renet_decoder_topk_workspace_bytes(M, N, K, k))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    _lib.check(L.renet_decoder_topk(P(x), P(w), P(b), P(col), P(begin), P(end), M, N, K, k, k, P(vals), P(idx), P(needed), P(ws),
                                    nbytes, _lib.stream()), 'renet_decoder_topk')
    assert int(needed.item()) > k
    small = decoder_topk(x, w, b, k, (col, begin, end), capacity=k)
    full = decoder_topk(x, w, b, k, (col, begin, end), capacity=N)
    dflt = decoder_topk(x, w, b, k, (col, begin, end))
    assert torch.equal(small[0], full[0]) and torch.equal(small[1], full[1])
    assert torch.equal(dflt[0], full[0]) and torch.equal(dflt[1], full[1])


def test_zero_rows():
    from renet_b200 import _lib
    from renet_b200.decoder import decoder_topk
    _, w, b = (t.to(DEV) for t in _fixture(1, 1000, 64, seed=1))
    x = torch.empty(0, 64, device=DEV)
    n0 = _lib.launch_count()
    v, i = decoder_topk(x, w, b, 10)
    assert v.shape == (0, 10) and i.shape == (0, 10) and i.dtype == torch.int64
    assert _lib.launch_count() == n0
