"""-m gpu: the decoder's training entries row by row against fp64.

renet_decoder_ce_fwd/_bwd (the hard-target loss of every training step: EPI 1 + ce_reduce_kernel, EPI 2 + the gradient
products) and renet_decoder_soft_ce_fwd/_bwd (the global model's soft targets: EPI 3 + soft_ce_reduce_kernel, EPI 4),
called through the C ABI, against one fp64 restatement of both losses: with T the target matrix (one-hot rows for hard
targets, P for soft ones), mass_i = sum_c T_ic and z = X W^T + b,
    lse_i = logsumexp_c z_ic,   loss_i = lse_i * mass_i - sum_c T_ic z_ic,   dz = g * (mass_i * softmax(z)_ic - T_ic),
    dX = dz W,   dW += dz^T X,   db += sum_i dz_i.
The inputs can show row and tile mistakes: rows at temperatures from 0.2 to 40, rows whose label beats every other logit
by 60, (forward only) rows around z = 80 where a sum of exponentials without the max subtracted overflows, and shapes at
the warpgroup (64 rows), unit (128 rows), half-tile (104 columns), tile (200 columns) and k-step (K % 8 == 4) edges.
Every output is judged per row (dX), per class row (dW) or per class (db), so a permuted or misread row cannot hide
behind the largest entry of the tensor; and every fixture first proves in fp64 that it sees the plausible bugs
(neighbour-row lse, lse + 0.01, softmax * 1.02, the last column tile dropped, P read with stride N) at 10x its bound.
dW and db accumulate onto a random base, dX starts as NaN, and sentinels after each gradient must survive: K % 8 == 4
once made the gradient products store past the end of each output row."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'

# Bounds of the per-row errors defined in _fwd_errors / _bwd_errors.  The worst errors measured on an H100 80GB HBM3
# (700 W power limit) over the shapes below are given beside each; the bounds leave a margin of 2.7x (forward) to 5x
# over them, and every mutant below misses them by at least 13x.
FWD_TOL = 2e-5     # loss and lse over max(1, max_c |z_ic|) (* max(1, mass_i) for the loss)            worst 7.4e-6
DX_TOL = 3e-4      # per row of dX, relative to the row's largest |entry| + the floor                      worst 9.0e-5
DW_TOL = 3e-4      # per class row of dW, likewise                                                          worst 7.1e-5
DB_TOL = 3e-4      # per class of db, relative to its |value| + the floor                                   worst 6.1e-5
PSUM_TOL = 1e-6    # psum_i relative                                                                        worst 1.2e-7
# The absolute floor of a gradient, as a fraction of the tensor's largest |entry|: rows whose gradient is almost 0
# (softmax ~ one-hot) are judged against it instead of against their own rounding noise.  db's is larger: each entry is
# one sum whose terms cancel for a class that is the label of rows that predict it well.
FLOOR = (1e-3, 1e-3, 1e-2)
MUTANT_FACTOR = 10.0

# (M, N, K): every M in {1, 64, 65, 128, 129, 1061}, N in {1, 103, 104, 105, 199, 200, 201, 23033} and K in
# {4, 12, 28, 400, 600} appears at least once; both passes run every shape
SHAPES = [(1, 23033, 600), (64, 201, 12), (65, 105, 28), (128, 1, 4), (129, 200, 400), (1061, 103, 12), (129, 104, 4),
          (65, 199, 400), (1061, 23033, 600)]
SOFT_SHAPES = [(1, 201, 600), (64, 104, 4), (65, 23033, 28), (128, 1, 12), (129, 199, 400), (1061, 7691, 400),
               (129, 105, 600), (65, 200, 12), (64, 103, 28)]


# ---- fixtures ---------------------------------------------------------------------------------------------------------------
def _inputs(M, N, K, seed, hot):
    """X [M, K], W [N, K], b [N] and a label per row.  Coordinates 0 and 1 of W are +s in one 'peak' class (N - 1 and
    N // 2) and -s elsewhere; rows 2, 7, 12, ... set one of them to 30 / s (temperature 1 otherwise), so their label (the
    peak class) beats every other logit by about 60.  With hot=True (the forward fixtures) row 0 is such a row too, and
    coordinate 2 of W is 1 and rows 4, 11, 18, ... set it to 78: logits around 80.  Every other row has its own
    temperature in [0.2, 40]."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=gen)
    w = torch.randn(N, K, generator=gen) * (0.12 / math.sqrt(K))
    b = torch.randn(N, generator=gen) * 2.0
    temp = torch.exp(torch.empty(M).uniform_(math.log(0.2), math.log(40.0), generator=gen))
    label = torch.randint(0, N, (M,), generator=gen)
    label[-1] = 0
    label[0] = N - 1                                   # M = 1 too: a label in the last column tile
    peak, s = (N - 1, N // 2), 0.25 / math.sqrt(K)   # s: about W's largest random entry, so that no coordinate of dX
    for j in range(2):                                # dwarfs the others
        w[:, j] = -s
        w[peak[j], j] = s
    peaked = torch.arange(M) % 5 == 2
    if hot:
        peaked[0] = True                               # the forward fixture's row 0 lives on its last-tile label
    hot_rows = (torch.arange(M) % 7 == 4) & ~peaked if hot else torch.zeros(M, dtype=torch.bool)
    temp[peaked | hot_rows] = 1.0
    x *= temp[:, None]
    x[:, :2] = 0.0
    for i in torch.nonzero(peaked).view(-1).tolist():
        j = (i // 5) % 2
        x[i, j] = 30.0 / s
        label[i] = peak[j]
    if hot:
        w[:, 2] = 1.0
        x[:, 2] = 0.0
        x[hot_rows, 2] = 78.0
    return x, w, b, label


def _soft_targets(M, N, label, gen):
    """Rows of P: 6 random columns, 2 in the last column tile and most of the mass on the row's label; every sixth row
    all zero; the last row's mass 1.7."""
    P = torch.zeros(M, N)
    last = (N - 1) // 200 * 200
    for i in range(M):
        cols = torch.cat((torch.randint(0, N, (6,), generator=gen), torch.randint(last, N, (2,), generator=gen)))
        P[i, cols] += torch.rand(8, generator=gen) + 0.05
        P[i, label[i]] += 4.0
        P[i] /= P[i].sum()
    P[torch.arange(M) % 6 == 3] = 0.0
    if M > 1:
        P[-1] *= 1.7
    return P


def _padded(P, pad=5):
    """P as a view [M, N] with row stride N + pad into a buffer whose pad columns hold 1e6."""
    M, N = P.shape
    buf = torch.full((M, N + pad), 1e6, device=P.device)
    buf[:, :N] = P
    return buf[:, :N], N + pad


# ---- the fp64 restatement and its mutants ---------------------------------------------------------------------------------
def _logits(x, w, b):
    z = x.double() @ w.double().t()
    return z + b.double() if b is not None else z


def _drop_start(N):
    """First column of the last work unit's half tile: the columns a kernel that skipped the last partial unit loses."""
    n0 = (N - 1) // 200 * 200
    return n0 + (104 if N - n0 > 104 else 0)


def _reference(z, T, g, mutant=None, T_mut=None):
    """(loss, lse, dz) in fp64 for logits z, targets T and gradient scale g; `mutant` names a plausible bug."""
    M, N = z.shape
    if mutant == 'P read with stride N':
        T = T_mut
    keep = torch.ones(N, dtype=torch.bool, device=z.device)
    if mutant == 'last column tile dropped':
        keep[_drop_start(N):] = False
    zk = z.masked_fill(~keep, float('-inf'))
    lse = torch.logsumexp(zk, 1)
    if mutant == 'neighbour-row lse':
        lse = lse.roll(1)
    elif mutant == 'lse + 0.01':
        lse = lse + 0.01
    mass = T.sum(1)
    sm = torch.exp(zk - lse[:, None])
    if mutant == 'softmax * 1.02':
        sm = sm * 1.02
        lse = lse + math.log(1.02)
    loss = lse * mass - (T * z).sum(1)
    dz = g * (mass[:, None] * sm - T)
    if mutant == 'last column tile dropped':
        dz[:, ~keep] = 0.0
    return loss, lse, dz


def _mutants(M, N, soft, backward):
    out = ['lse + 0.01', 'softmax * 1.02']
    if M > 1:
        out.append('neighbour-row lse')            # one row has no neighbour, and its stride is never used
        if soft and N > 1:                         # N = 1: loss and gradient are 0 whatever P holds
            out.append('P read with stride N')
    if N > 1 or not backward:
        out.append('last column tile dropped')     # N = 1: every gradient is 0 with its only column or without it
    return out


def _nan_inf(t):
    return torch.nan_to_num(t, nan=float('inf'))


def _fwd_errors(loss, lse, z, mass, ref_loss, ref_lse):
    """max over rows of |loss_i - ref| / (max(1, max_c |z_ic|) * max(1, mass_i)) and |lse_i - ref| / max(1, max_c |z_ic|)."""
    zs = z.abs().amax(1).clamp(min=1.0)
    e_loss = _nan_inf((loss.double() - ref_loss).abs() / (zs * mass.clamp(min=1.0)))
    e_lse = _nan_inf((lse.double() - ref_lse).abs() / zs)
    return float(torch.maximum(e_loss, e_lse).max())


def _per_row(a, r, floor_frac):
    """max_i max_j |a_ij - r_ij| / (max_j |r_ij| + floor_frac * max |r|)."""
    r = r.view(r.shape[0], -1)
    a = a.double().view(r.shape)
    floor = floor_frac * float(r.abs().max()) + 1e-300
    return float(_nan_inf((a - r).abs().amax(1) / (r.abs().amax(1) + floor)).max())


def _grads(dz, x, w):
    return dz @ w.double(), dz.t() @ x.double(), dz.sum(0)


def _bwd_errors(got, ref):
    return tuple(_per_row(a, r, f) for a, r, f in zip(got, ref, FLOOR))


# ---- the C ABI --------------------------------------------------------------------------------------------------------------
def _guarded(values, tail=64):
    """A tensor shaped like `values` (a copy) followed in memory by `tail` sentinel floats: (view, tail view)."""
    buf = torch.full((values.numel() + tail,), -7.25e7, device=DEV)
    buf[:values.numel()] = values.reshape(-1)
    return buf[:values.numel()].view(values.shape), buf[values.numel():]


def _ce_fwd(x, w, b, label):
    from renet_b200 import _lib
    L, P = _lib.lib(), _lib.ptr
    M, K = x.shape
    N = w.shape[0]
    loss, lse = torch.full((M,), float('nan'), device=DEV), torch.full((M,), float('nan'), device=DEV)
    nbytes = int(L.renet_decoder_ce_workspace_bytes(M, N, K))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    _lib.check(L.renet_decoder_ce_fwd(P(x), P(w), P(b), P(label), P(loss), P(lse), M, N, K, P(ws), nbytes, _lib.stream()),
               'renet_decoder_ce_fwd')
    return loss, lse


def _soft_fwd(x, w, b, Pv, ldp):
    from renet_b200 import _lib
    L, P = _lib.lib(), _lib.ptr
    M, K = x.shape
    N = w.shape[0]
    loss, lse, psum = (torch.full((M,), float('nan'), device=DEV) for _ in range(3))
    nbytes = int(L.renet_decoder_soft_ce_workspace_bytes(M, N, K))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    _lib.check(L.renet_decoder_soft_ce_fwd(P(x), P(w), P(b), P(Pv), ldp, P(loss), P(lse), P(psum), M, N, K, P(ws), nbytes,
                                           _lib.stream()), 'renet_decoder_soft_ce_fwd')
    return loss, lse, psum


def _bwd(x, w, b, lse, scale, d_scale, dw0, db0, label=None, soft=None):
    """renet_decoder_ce_bwd (label) or renet_decoder_soft_ce_bwd (soft = (P view, ldp, psum)): dX starts as NaN, dW and db
    (None: NULL) as copies of dw0 / db0, each followed by sentinels that must survive.  Returns (dX, dW, db)."""
    from renet_b200 import _lib
    L, P = _lib.lib(), _lib.ptr
    M, K = x.shape
    N = w.shape[0]
    dX, tX = _guarded(torch.full((M, K), float('nan'), device=DEV))
    dW, tW = _guarded(dw0)
    db, tb = _guarded(db0) if db0 is not None else (None, None)
    if soft is None:
        nbytes = int(L.renet_decoder_ce_bwd_workspace_bytes(M, N, K))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        rc = L.renet_decoder_ce_bwd(P(x), P(w), P(b), P(label), P(lse), scale, P(d_scale), P(dX), P(dW), P(db), M, N, K, P(ws),
                                    nbytes, _lib.stream())
    else:
        Pv, ldp, psum = soft
        nbytes = int(L.renet_decoder_soft_ce_bwd_workspace_bytes(M, N, K))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        rc = L.renet_decoder_soft_ce_bwd(P(x), P(w), P(b), P(Pv), ldp, P(lse), P(psum), scale, P(d_scale), P(dX), P(dW), P(db),
                                         M, N, K, P(ws), nbytes, _lib.stream())
    _lib.check(rc, 'renet_decoder_soft_ce_bwd' if soft is not None else 'renet_decoder_ce_bwd')
    for t in (tX, tW, tb):
        if t is not None:
            assert bool((t == -7.25e7).all()), 'a gradient was written past its end'
    return dX, dW, db


def _base(ref):
    """The accumulated gradients' starting value: random, 1e-2 of the gradient's size (lost, it fails the bound by far;
    rounded with the gradient to fp32, it stays far below the floor)."""
    gen = torch.Generator(device=DEV).manual_seed(ref.numel())
    return (torch.randn(ref.shape, device=DEV, generator=gen, dtype=torch.float64) * 1e-2 * float(ref.abs().max())).float()


def _device(*ts):
    return [t.to(DEV) if t is not None else None for t in ts]


def _check_mutants(name, errs_of, bounds, mutants):
    """Every mutant misses every bound by MUTANT_FACTOR; returns the smallest mutant error / bound."""
    weakest = float('inf')
    for m in mutants:
        ratios = [e / t for e, t in zip(errs_of(m), bounds)]
        assert min(ratios) >= MUTANT_FACTOR, ('the fixture cannot see the bug', name, m, ratios)
        weakest = min(weakest, min(ratios))
    return weakest


# ---- hard targets -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('M,N,K', SHAPES)
def test_ce_forward_per_row_vs_fp64(M, N, K):
    x, w, b, label = _device(*_inputs(M, N, K, seed=M * 31 + N + K, hot=True))
    z = _logits(x, w, b)
    T = torch.nn.functional.one_hot(label, N).double()
    mass = T.sum(1)
    ref_loss, ref_lse, _ = _reference(z, T, 1.0)
    weakest = _check_mutants('ce fwd', lambda m: (_fwd_errors(*_reference(z, T, 1.0, m)[:2], z, mass, ref_loss, ref_lse),),
                             (FWD_TOL,), _mutants(M, N, False, False))
    loss, lse = _ce_fwd(x, w, b, label.int())
    err = _fwd_errors(loss, lse, z, mass, ref_loss, ref_lse)
    print('ce fwd M=%d N=%d K=%d: max|z| %.1f, error / bound %.3g, weakest mutant / bound %.3g'
          % (M, N, K, float(z.abs().max()), err / FWD_TOL, weakest))
    assert err <= FWD_TOL


@pytest.mark.parametrize('M,N,K', SHAPES)
def test_ce_backward_per_row_vs_fp64(M, N, K):
    x, w, b, label = _device(*_inputs(M, N, K, seed=M * 37 + N + K, hot=False))
    z = _logits(x, w, b)
    T = torch.nn.functional.one_hot(label, N).double()
    scale, d_scale = 1.0 / M, torch.tensor([0.7], device=DEV)
    g = scale * 0.7
    ref = _grads(_reference(z, T, g)[2], x, w)
    bounds = (DX_TOL, DW_TOL, DB_TOL)
    weakest = _check_mutants('ce bwd', lambda m: _bwd_errors(_grads(_reference(z, T, g, m)[2], x, w), ref), bounds,
                             _mutants(M, N, False, True))
    _, lse = _ce_fwd(x, w, b, label.int())
    dw0, db0 = _base(ref[1]), _base(ref[2])
    dX, dW, db = _bwd(x, w, b, lse, scale, d_scale, dw0, db0, label=label.int())
    got = (dX, dW.double() - dw0.double(), db.double() - db0.double())
    errs = _bwd_errors(got, ref)
    print('ce bwd M=%d N=%d K=%d: max|z| %.1f, error / bound dX %.3g dW %.3g db %.3g, weakest mutant / bound %.3g'
          % ((M, N, K, float(z.abs().max())) + tuple(e / t for e, t in zip(errs, bounds)) + (weakest,)))
    for e, t, nm in zip(errs, bounds, ('dX', 'dW', 'db')):
        assert e <= t, (nm, e)


# ---- soft targets -----------------------------------------------------------------------------------------------------------
def _soft_fixture(M, N, K, seed, hot):
    x, w, b, label = _inputs(M, N, K, seed, hot)
    P = _soft_targets(M, N, label, torch.Generator().manual_seed(seed + 1))
    x, w, b, P = _device(x, w, b, P)
    Pv, ldp = _padded(P)
    P_stride_n = Pv.as_strided((M, N), (N, 1)).double()       # what a kernel that ignored ldp would read
    return x, w, b, Pv, ldp, P.double(), P_stride_n


@pytest.mark.parametrize('M,N,K', SOFT_SHAPES)
def test_soft_ce_forward_per_row_vs_fp64(M, N, K):
    x, w, b, Pv, ldp, T, T_n = _soft_fixture(M, N, K, seed=M * 41 + N + K, hot=True)
    z = _logits(x, w, b)
    mass = T.sum(1)
    ref_loss, ref_lse, _ = _reference(z, T, 1.0)
    weakest = _check_mutants('soft fwd', lambda m: (_fwd_errors(*_reference(z, T, 1.0, m, T_n)[:2], z, mass, ref_loss, ref_lse),),
                             (FWD_TOL,), _mutants(M, N, True, False))
    loss, lse, psum = _soft_fwd(x, w, b, Pv, ldp)
    err = _fwd_errors(loss, lse, z, mass, ref_loss, ref_lse)
    zero = mass == 0
    assert bool((loss[zero] == 0).all()) and bool((psum[zero] == 0).all())        # zero-mass rows: exactly 0
    e_psum = float(((psum.double() - mass).abs() / mass.clamp(min=1e-30)).max())
    print('soft fwd M=%d N=%d K=%d: max|z| %.1f, error / bound %.3g, psum %.3g, weakest mutant / bound %.3g'
          % (M, N, K, float(z.abs().max()), err / FWD_TOL, e_psum / PSUM_TOL, weakest))
    assert err <= FWD_TOL
    assert e_psum <= PSUM_TOL


@pytest.mark.parametrize('M,N,K', SOFT_SHAPES)
def test_soft_ce_backward_per_row_vs_fp64(M, N, K):
    x, w, b, Pv, ldp, T, T_n = _soft_fixture(M, N, K, seed=M * 43 + N + K, hot=False)
    z = _logits(x, w, b)
    scale, d_scale = 1.0 / M, torch.tensor([0.7], device=DEV)
    g = scale * 0.7
    ref = _grads(_reference(z, T, g)[2], x, w)
    bounds = (DX_TOL, DW_TOL, DB_TOL)
    weakest = _check_mutants('soft bwd', lambda m: _bwd_errors(_grads(_reference(z, T, g, m, T_n)[2], x, w), ref), bounds,
                             _mutants(M, N, True, True))
    _, lse, psum = _soft_fwd(x, w, b, Pv, ldp)
    dw0, db0 = _base(ref[1]), _base(ref[2])
    dX, dW, db = _bwd(x, w, b, lse, scale, d_scale, dw0, db0, soft=(Pv, ldp, psum))
    got = (dX, dW.double() - dw0.double(), db.double() - db0.double())
    errs = _bwd_errors(got, ref)
    zero = T.sum(1) == 0
    assert bool((dX[zero] == 0).all())                                            # zero-mass rows: exactly 0
    print('soft bwd M=%d N=%d K=%d: max|z| %.1f, error / bound dX %.3g dW %.3g db %.3g, weakest mutant / bound %.3g'
          % ((M, N, K, float(z.abs().max())) + tuple(e / t for e, t in zip(errs, bounds)) + (weakest,)))
    for e, t, nm in zip(errs, bounds, ('dX', 'dW', 'db')):
        assert e <= t, (nm, e)


# ---- the optional arguments -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('soft', [False, True])
def test_null_d_scale_is_one(soft):
    """d_scale = NULL gives bitwise what a device scalar holding 1.0 gives."""
    M, N, K = 129, 201, 28
    x, w, b, label = _device(*_inputs(M, N, K, seed=3, hot=False))
    dw0, db0 = torch.randn(N, K, device=DEV), torch.randn(N, device=DEV)
    if soft:
        Pv, ldp = _padded(_soft_targets(M, N, label.cpu(), torch.Generator().manual_seed(4)).to(DEV))
        _, lse, psum = _soft_fwd(x, w, b, Pv, ldp)
        kw = dict(soft=(Pv, ldp, psum))
    else:
        _, lse = _ce_fwd(x, w, b, label.int())
        kw = dict(label=label.int())
    one = _bwd(x, w, b, lse, 1.0 / M, torch.ones(1, device=DEV), dw0, db0, **kw)
    null = _bwd(x, w, b, lse, 1.0 / M, None, dw0, db0, **kw)
    for a, c in zip(one, null):
        assert torch.equal(a, c)


@pytest.mark.parametrize('soft', [False, True])
def test_null_bias(soft):
    """bias = NULL computes what a zero bias computes, bit for bit: the loss rows and lse, and dX and dW with dbias = NULL;
    with dbias given, db is the zero bias's db."""
    M, N, K = 65, 1001, 12
    x, w, _, label = _device(*_inputs(M, N, K, seed=5, hot=False))
    zero = torch.zeros(N, device=DEV)
    dw0, db0 = torch.randn(N, K, device=DEV), torch.randn(N, device=DEV)
    if soft:
        Pv, ldp = _padded(_soft_targets(M, N, label.cpu(), torch.Generator().manual_seed(6)).to(DEV))
        fz, fn = _soft_fwd(x, w, zero, Pv, ldp), _soft_fwd(x, w, None, Pv, ldp)
        kw = dict(soft=(Pv, ldp, fz[2]))
    else:
        fz, fn = _ce_fwd(x, w, zero, label.int()), _ce_fwd(x, w, None, label.int())
        kw = dict(label=label.int())
    for a, c in zip(fz, fn):
        assert torch.equal(a, c)
    lse = fz[1]
    with_zero = _bwd(x, w, zero, lse, 1.0 / M, None, dw0, db0, **kw)
    without = _bwd(x, w, None, lse, 1.0 / M, None, dw0, None, **kw)
    assert torch.equal(with_zero[0], without[0]) and torch.equal(with_zero[1], without[1])
    db_only = _bwd(x, w, None, lse, 1.0 / M, None, dw0, db0, **kw)
    assert torch.equal(db_only[2], with_zero[2])


def test_zero_rows_write_nothing():
    """M = 0 returns success at once from all four entries and leaves every output as it was."""
    from renet_b200 import _lib
    L, P = _lib.lib(), _lib.ptr
    N, K = 201, 12
    x, w, b, label = _device(*_inputs(1, N, K, seed=7, hot=False))
    out = torch.full((4 * N * K,), 3.5, device=DEV)
    o = P(out)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    s = _lib.stream()
    assert L.renet_decoder_ce_fwd(P(x), P(w), P(b), P(label), o, o, 0, N, K, P(ws), 1 << 20, s) == 0
    assert L.renet_decoder_ce_bwd(P(x), P(w), P(b), P(label), o, 1.0, None, o, o, o, 0, N, K, P(ws), 1 << 20, s) == 0
    assert L.renet_decoder_soft_ce_fwd(P(x), P(w), P(b), o, N, o, o, o, 0, N, K, P(ws), 1 << 20, s) == 0
    assert L.renet_decoder_soft_ce_bwd(P(x), P(w), P(b), o, N, o, o, 1.0, None, o, o, o, 0, N, K, P(ws), 1 << 20, s) == 0
    torch.cuda.synchronize()
    assert bool((out == 3.5).all())
