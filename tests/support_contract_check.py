"""The training step's support kernels per element against float64 or an exact restatement, with the serving kernels
asserted (cases for tests/test_gpu_support_contract.py; importing this module needs no GPU).

U = 2^-24.  Every case builds its inputs explicitly and asserts on the host the property it exists for before it launches.

Entry points, references and bars
  renet_grad_sumsq      fp64 sum of g^2.  Bar (L + 24) U sum g^2, L = the most terms one thread adds: 4 per float4 pass of
                        the 592 x 256 partial grid, + 1 for the scalar tail of block 0; 24 covers the reduction tree (5 shuffle
                        levels + 7 warp partials in a block, 5 + 5 levels in the final block, 1 for accumulate / the last add).
                        With accumulate = 1 the base is added: + U |base + sum|.
  renet_adam_step       one fp64 step of clip + torch.optim.Adam(amsgrad=False) from the kernel's own fp32 state (p, m, v)
                        before the step, with the hyper-parameters rounded to fp32 as the kernel sees them and the clip factor
                        from the kernel's sumsq.  Bar per element C_ADAM U times the size of its terms:
                          Tg = |g gs clip| + |wd p|,  Tm = b1 |m| + (1 - b1) Tg,  Tv = b2 v + (1 - b2) Tg^2,
                          m: C_ADAM U Tm;  v: C_ADAM U Tv;  p: C_ADAM U (|p| + |step| + lr/bc1 Tm / denom).
                        Counting roundings: the clip coefficient 5, g' 1 more, m' <= 8 U Tm, v' <= 15 U Tv, the denominator
                        <= 11 U relative, the step 4 more, the update 1: C_ADAM = 16 holds by construction.
  renet_scatter_add_rows  default mode: fp64 base + sum of the rows, bar (n_t + 1) U (|base| + sum |src|) per element,
                        n_t = the rows sent to that target; deterministic mode: EXACT, numpy fp32 acc = 0; acc += src[j] in
                        ascending source row, then base + acc, and two runs bitwise equal.
  renet_segment_pool_fwd/_bwd  max, argmax (first maximum wins) and both backwards exact; mean forward exact against the
                        numpy fp32 sequential sum in row order divided by float(n).  Rows of dH outside every argmax are 0.
  renet_selfloop_gemm_bwd  fp64 dLoop @ Wloop^T and base + H[h_index]^T @ dLoop; bar (K + 4) U sum |a b| per element (|base|
                        included), as in the GEMM suite.
  renet_dropout_mask    EXACT against a numpy Philox4x32-10 (restated from the algorithm, checked against Random123's known
                        answer and curand's constants by tests/test_philox_restatement.py): scale = 1/(1-p) in fp32 when
                        (float)w * 2^-32 >= p, else 0.  renet_gru_fwd_dropout's materialised X4d / X3d (the forward workspace)
                        must equal the gathered inputs times these masks, with X3 elements at S*4h + i*3h + c.
  renet_build_csr, renet_readout_subgraph, renet_induce_edges  EXACT against numpy restatements of the header contracts;
                        every output is over-allocated with sentinels past its valid length, and they must survive.

The GRU dropout backward in deterministic mode (ld = 4h, the seq_s / seq_r indirection) is checked through d_ent / d_rel:
the scatter bar against the fp64 sum of the kernel's own dX4 column blocks (located at the end of the backward
workspace, gru.cu's carve_bwd), the exact sequential restatement over them, and two runs bitwise equal.

Which kernel ran: every case names the kernels it expects; the call is repeated under torch.profiler (CUDA activities, a
call of its own) and the set of kernel names (template booleans kept, CUB's radix sort / scan kernels as 'cub') must be
exactly that set.  Cases whose path depends on deterministic mode run in both modes, switched through
torch.use_deterministic_algorithms and restored afterwards."""
import contextlib
import functools
import re

import numpy as np
import torch

DEV = 'cuda:0'
U = 2.0 ** -24
C_ADAM = 16.0
SUMSQ_THREADS, SUMSQ_BLOCKS = 256, 592
ADAM_CAP = 132 * 8 * 256 * 4               # floats one pass of the Adam grid covers: 1 081 344
EXTRA = 8                                  # sentinel elements past every output
SENT_I, SENT_F = -7, 1234.5
WORST = {}                                 # label -> (largest err / bound, case, what)


# ---- plumbing ---------------------------------------------------------------------------------------------------------------
def lib():
    from renet_b200 import _lib
    return _lib, _lib.lib(), _lib.ptr


@contextlib.contextmanager
def deterministic(on):
    _lib, L, _ = lib()
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        _lib.stream()
        assert L.renet_get_deterministic() == int(on)
        yield
    finally:
        torch.use_deterministic_algorithms(before)
        _lib.stream()


def short_name(name):
    """'cub' for CUB's kernels, else the kernel's bare name with its template booleans: segment_pool_fwd_kernel<true>"""
    if 'cub::' in name:
        return 'cub'
    n = name[5:] if name.startswith('void ') else name
    n = n.replace('(anonymous namespace)::', '')
    m = re.match(r'(?:\w+::)*(\w+)', n)
    base, rest = m.group(1), n[m.end():]
    flags = []
    if rest.startswith('<'):
        depth = 0
        for j, ch in enumerate(rest):
            depth += ch == '<'
            depth -= ch == '>'
            if depth == 0:
                break
        flags = ['true' if f in ('true', '(bool)1') else 'false' for f in re.findall(r'true|false|\(bool\)[01]', rest[1:j])]
    return base + ('<%s>' % ','.join(flags) if flags else '')


def kernels_of(fn, want=()):
    """the union of the kernel names over up to 10 traces of fn, stopping once it holds every name in want (or
    want(union) holds, for a callable).  A trace can lose the record of a kernel that did run (seen with the first kernel
    of a call), never invent one, and every call launches the same kernels: so the union is what fn launches, and only
    a kernel that never shows in any trace fails.  In a process that has run many traces records go missing most often at
    the edges of a trace, so each trace calls fn twice between two torch kernels (not counted)."""
    seen = set()
    prime = torch.zeros(1, device=DEV)
    for _ in range(10):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            prime.add_(1)
            torch.cuda.synchronize()
            fn()
            fn()
            torch.cuda.synchronize()
            prime.add_(1)
            torch.cuda.synchronize()
        seen |= {short_name(ev.name) for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and
                 not ev.name.startswith(('Memset', 'Memcpy')) and 'at::' not in ev.name}
        if (want(seen) if callable(want) else set(want) <= seen):
            break
    return seen


def assert_kernels(case, fn, expected):
    seen = kernels_of(fn, expected)
    assert seen == set(expected), '%s: ran %s, expected %s' % (case, sorted(seen), sorted(expected))


def note(label, case, what, ratio):
    if ratio > WORST.get(label, (-1.0,))[0]:
        WORST[label] = (ratio, case, what)


def check_bound(label, case, what, got, ref, bound):
    """|got - ref| <= bound per element (float64 tensors on the device); bound 0 means exact"""
    assert torch.isfinite(got).all(), (case, what, 'not finite')
    err = (got.double() - ref).abs()
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, float('inf'), 0.0).double())
    worst = float(ratio.max()) if ratio.numel() else 0.0
    note(label, case, what, worst)
    i = int(ratio.flatten().argmax()) if ratio.numel() else 0
    assert worst <= 1.0, '%s %s (%s): element %d is %.3g x its bound off (got %r, ref %r); %d elements fail' % (
        case, what, label, i, worst, float(got.flatten()[i]), float(ref.flatten()[i]), int((ratio > 1).sum()))


def exact(label, case, what, got, ref):
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, (case, what, got.shape, ref.shape)
    same = (got == ref) | (np.isnan(got) & np.isnan(ref)) if got.dtype.kind == 'f' else got == ref
    if got.dtype.kind == 'f':
        same &= np.signbit(got) == np.signbit(ref)
    bad = np.flatnonzero(~same.reshape(-1))
    note(label, case, what, 0.0 if bad.size == 0 else float('inf'))
    assert bad.size == 0, '%s %s (%s): %d elements differ, first at %d: got %r, expected %r' % (
        case, what, label, bad.size, bad[0], got.reshape(-1)[bad[0]], ref.reshape(-1)[bad[0]])


def i32(a, extra=0):
    t = torch.full((len(a) + extra,), SENT_I, dtype=torch.int32)
    t[:len(a)] = torch.from_numpy(np.asarray(a, dtype=np.int32))
    return t.to(DEV)


def cpu(t):
    return t.detach().cpu().numpy()


CASES = {}


def case(name):
    def reg(fn):
        assert name not in CASES, name
        CASES[name] = functools.partial(fn, name)
        return fn
    return reg


# ---- renet_grad_sumsq / renet_adam_step ------------------------------------------------------------------------------------
def sumsq_terms(n):
    """(blocks of the partial kernel, L = the most terms one thread adds)"""
    n4 = n // 4
    want = (n4 + SUMSQ_THREADS - 1) // SUMSQ_THREADS
    nblk = 0 if n == 0 else min(max(want, 1), SUMSQ_BLOCKS)
    passes = -(-n4 // (nblk * SUMSQ_THREADS)) if n4 else 0
    return nblk, 4 * passes + (1 if n % 4 else 0)


def adam_passes(n):
    n4 = n // 4
    grid = min(max((n4 + 255) // 256, 1), 132 * 8)
    return -(-n4 // (grid * 256)) if n4 else 0


def run_sumsq(cs, g, accumulate=0, base=0.0):
    _lib, L, P = lib()
    n = g.numel()
    ws = torch.full((int(L.renet_grad_sumsq_workspace_bytes()) // 4,), float('nan'), device=DEV)
    out = torch.full((1 + EXTRA,), SENT_F, device=DEV)

    def call():
        out[0] = base
        _lib.check(L.renet_grad_sumsq(P(g), n, P(out), accumulate, P(ws), ws.numel() * 4, _lib.stream()), 'grad_sumsq')
        return out

    nblk, Lt = sumsq_terms(n)
    n0 = _lib.launch_count()
    call()
    assert _lib.launch_count() - n0 == (2 if nblk else 1), (cs, 'grad_sumsq launch count')
    s = float(out[0])
    ref = float((g.double() ** 2).sum())
    b = float(np.float32(base)) if accumulate else 0.0
    bound = (Lt + 24) * U * ref + (U * abs(b + ref) if accumulate else 0.0)
    check_bound('grad_sumsq', cs, 'sumsq', torch.tensor([s], dtype=torch.float64), torch.tensor([b + ref], dtype=torch.float64),
                torch.tensor([bound], dtype=torch.float64))
    assert torch.equal(out[1:], torch.full((EXTRA,), SENT_F, device=DEV)), (cs, 'sumsq wrote past out[0]')
    assert_kernels(cs, call, {'grad_sumsq_final_kernel'} | ({'grad_sumsq_partial_kernel'} if nblk else set()))
    again = call()
    assert float(again[0]) == s, (cs, 'sumsq not reproducible')
    return out[:1].clone()


def run_adam(cs, n, step=1, gs=1.0, max_norm=1.0, wd=1e-5, use_sumsq=True, gscale=3.0, seed=0, lr=1e-3):
    _lib, L, P = lib()
    gen = torch.Generator(device=DEV).manual_seed(seed)
    pad = (-n) % 4 + 4
    buf = lambda: torch.empty(n + pad, device=DEV)
    p0 = torch.randn(n, device=DEV, generator=gen)
    g = buf()[:n]
    g.copy_(torch.randn(n, device=DEV, generator=gen) * gscale)
    m0 = torch.randn(n, device=DEV, generator=gen) * 1e-2
    v0 = torch.rand(n, device=DEV, generator=gen) ** 2 * 1e-3
    sumsq = run_sumsq(cs, g) if use_sumsq else None
    tails = [buf() for _ in range(3)]
    for t in tails:
        t[n:] = SENT_F
    p, m, v = (t[:n] for t in tails)

    def call():
        p.copy_(p0), m.copy_(m0), v.copy_(v0)
        _lib.check(L.renet_adam_step(P(p), P(g), P(m), P(v), n, lr, 0.9, 0.999, 1e-8, wd, step, P(sumsq), max_norm, gs,
                                     _lib.stream()), 'adam_step')

    n0 = _lib.launch_count()
    call()
    assert _lib.launch_count() - n0 == 1, (cs, 'adam_step launch count')
    for t in tails:
        assert torch.equal(t[n:], torch.full_like(t[n:], SENT_F)), (cs, 'adam wrote past n')
    assert_kernels(cs, call, {'adam_step_kernel'})
    clip = clip_coef(float(sumsq[0]), max_norm, gs) if use_sumsq and max_norm > 0 else 1.0
    (P1, M1, V1), (bp, bm, bv) = adam_ref(p0, g, m0, v0, step, clip, lr, 0.9, 0.999, 1e-8, wd, gs)
    check_bound('adam m', cs, 'm', m, M1, bm)
    check_bound('adam v', cs, 'v', v, V1, bv)
    check_bound('adam p', cs, 'p', p, P1, bp)
    return clip


def f32(x):
    return float(np.float32(x))


def clip_coef(sumsq, max_norm, gs=1.0):
    """renet_adam_step's clip factor from a sum of squares: clip_grad_norm_'s max_norm / (|g| + 1e-6), capped at 1"""
    return min(1.0, f32(max_norm) / (np.sqrt(sumsq) * f32(gs) + 1e-6))


def adam_ref(p0, g, m0, v0, step, clip, lr, b1, b2, eps, wd, gs=1.0):
    """one fp64 step of torch.optim.Adam(amsgrad=False) with weight decay on the clipped gradient g * gs * clip, the
    hyper-parameters rounded to fp32 as the kernel sees them -> ((p, m, v), (their bounds)), as the module docstring derives"""
    lr_, b1, b2, eps, wd_, gs_ = f32(lr), f32(b1), f32(b2), f32(eps), f32(wd), f32(gs)
    bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step
    P0, G, M0, V0 = p0.double(), g.double(), m0.double(), v0.double()
    ga = G * gs_ * clip
    gg = ga + wd_ * P0
    Tg = ga.abs() + (wd_ * P0).abs()
    M1 = b1 * M0 + (1 - b1) * gg
    V1 = b2 * V0 + (1 - b2) * gg * gg
    denom = V1.sqrt() / np.sqrt(bc2) + eps
    stp = lr_ / bc1 * M1 / denom
    P1 = P0 - stp
    Tm = b1 * M0.abs() + (1 - b1) * Tg
    Tv = b2 * V0 + (1 - b2) * Tg * Tg
    return (P1, M1, V1), (C_ADAM * U * (P0.abs() + stp.abs() + lr_ / bc1 * Tm / denom), C_ADAM * U * Tm, C_ADAM * U * Tv)


for _n in (1, 3, 4, 5, 1023):
    @case('adam-n%d' % _n)
    def _(cs, n=_n):
        assert n < 4 * 256 or n == 1023
        assert run_adam(cs, n, gscale=30.0) < 1.0 or n < 4            # clipped wherever the norm can exceed 1


@case('adam-loop-cap-minus-1')
def _(cs):
    n = ADAM_CAP - 1
    assert adam_passes(n) == 1 and n % 4 == 3
    run_adam(cs, n, step=2, gs=0.5)


@case('adam-loop-cap-plus-1')
def _(cs):
    n = ADAM_CAP + 1
    assert adam_passes(n) == 1 and n % 4 == 1, 'one full pass, then the scalar tail'
    assert run_adam(cs, n, step=2, gs=0.5) < 1.0


@case('adam-loop-cap-plus-4')
def _(cs):
    n = ADAM_CAP + 4
    assert adam_passes(n) == 2, 'n > 1 081 344 (one float4 more): the Adam loop runs twice'
    run_adam(cs, n, step=2, gs=0.125)


@case('adam-loop-2cap-plus-3-unclipped')
def _(cs):
    n = 2 * ADAM_CAP + 3
    assert adam_passes(n) == 2 and n % 4 == 3
    assert run_adam(cs, n, step=10, gs=0.125, gscale=1e-5) == 1.0


@case('adam-flat-20.2M')
def _(cs):
    n = 20_200_003
    assert adam_passes(n) == 19 and sumsq_terms(n)[0] == SUMSQ_BLOCKS
    run_adam(cs, n, step=3)


@case('adam-step-10000-gs-0.125')
def _(cs):
    assert run_adam(cs, 4099, step=10000, gs=0.125, gscale=300.0) < 1.0


@case('adam-no-clip-null-sumsq')
def _(cs):
    run_adam(cs, 100003, step=2, gs=0.5, max_norm=0.0, use_sumsq=False)


@case('adam-max-norm-0-with-sumsq')
def _(cs):
    run_adam(cs, 5001, max_norm=0.0, gscale=30.0)


@case('adam-weight-decay-0')
def _(cs):
    run_adam(cs, 70001, wd=0.0, step=2)


@case('adam-zero-grads')
def _(cs):
    assert run_adam(cs, 4097, gscale=0.0, wd=0.0) == 1.0


@case('adam-n0')
def _(cs):
    _lib, L, P = lib()
    t = torch.full((4,), SENT_F, device=DEV)
    assert_kernels(cs, lambda: _lib.check(L.renet_adam_step(P(t), P(t), P(t), P(t), 0, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, None, 0.0,
                                                            1.0, _lib.stream()), 'adam n=0'), set())
    assert torch.equal(t, torch.full((4,), SENT_F, device=DEV))


for _n in (1, 3, 4, 5, 1023, ADAM_CAP - 1, ADAM_CAP + 1, 2 * ADAM_CAP + 3, 20_200_003):
    @case('sumsq-n%d' % _n)
    def _(cs, n=_n):
        gen = torch.Generator(device=DEV).manual_seed(n)
        g = torch.empty(n + 4, device=DEV)[:n]
        g.copy_(torch.randn(n, device=DEV, generator=gen))
        nblk, Lt = sumsq_terms(n)
        if n > 4 * SUMSQ_THREADS * SUMSQ_BLOCKS:
            assert Lt > 4, 'the partial loop runs more than once'
        run_sumsq(cs, g)

for _acc in (0, 1):
    @case('sumsq-accumulate-%d' % _acc)
    def _(cs, acc=_acc):
        g = torch.randn(300007, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
        run_sumsq(cs, g, accumulate=acc, base=12345.678)

    @case('sumsq-n0-accumulate-%d' % _acc)
    def _(cs, acc=_acc):
        # n = 0 with a valid workspace: only the final kernel runs; out = 0, or the base with accumulate
        _lib, L, P = lib()
        ws = torch.full((int(L.renet_grad_sumsq_workspace_bytes()) // 4,), float('nan'), device=DEV)
        g = torch.full((4,), SENT_F, device=DEV)
        out = torch.full((2,), SENT_F, device=DEV)

        def call():
            out[0] = 7.25
            _lib.check(L.renet_grad_sumsq(P(g), 0, P(out), acc, P(ws), ws.numel() * 4, _lib.stream()), 'grad_sumsq n=0')

        n0 = _lib.launch_count()
        call()
        assert _lib.launch_count() - n0 == 1, (cs, 'n = 0 must launch the final kernel only')
        assert float(out[0]) == (7.25 if acc else 0.0) and float(out[1]) == SENT_F, (cs, cpu(out))
        assert torch.isnan(ws).all(), (cs, 'n = 0 wrote the workspace')
        assert_kernels(cs, call, {'grad_sumsq_final_kernel'})


# ---- renet_scatter_add_rows ------------------------------------------------------------------------------------------------
def seq_scatter(base, src, index):
    """numpy fp32: per target acc = 0; acc += src[j] in ascending source row; base + acc"""
    out = base.copy()
    if len(index) == 0:
        return out
    order = np.argsort(index, kind='stable')
    keys = index[order]
    starts = np.flatnonzero(np.concatenate(([True], keys[1:] != keys[:-1])))
    sizes = np.diff(np.concatenate((starts, [len(keys)])))
    acc = np.zeros((len(starts), src.shape[1]), dtype=np.float32)
    for k in range(int(sizes.max())):
        live = np.flatnonzero(sizes > k)
        acc[live] += src[order[starts[live] + k]]
    out[keys[starts]] += acc
    return out


def scatter_kernels(det, vec):
    if det:
        return {'scatter_keys_kernel', 'cub', 'scatter_add_rows_sorted_kernel'}
    return {'scatter_add_rows_kernel'} if vec else {'scatter_add_rows_scalar_kernel'}


def run_scatter(cs, index, T, d, det, dst_shift=0, seed=0):
    _lib, L, P = lib()
    gen = torch.Generator(device=DEV).manual_seed(seed)
    index = np.asarray(index, dtype=np.int64)
    n = len(index)
    src = torch.randn(max(n, 1), d, device=DEV, generator=gen)[:n]
    base = torch.randn(T, d, device=DEV, generator=gen)
    flat = torch.empty(T * d + dst_shift + EXTRA, device=DEV)
    dst = flat[dst_shift:dst_shift + T * d].view(T, d)
    vec = d % 4 == 0 and dst_shift % 4 == 0
    assert (dst.data_ptr() % 16 == 0) == (dst_shift % 4 == 0)
    idx = i32(index, 1)

    def call():
        flat.fill_(SENT_F)
        dst.copy_(base)
        _lib.check(L.renet_scatter_add_rows(P(src) if n else P(base), P(idx), P(dst), n, d, _lib.stream()), 'scatter_add_rows')
        return dst.clone()

    with deterministic(det):
        got = call()
        assert torch.equal(flat[:dst_shift], torch.full((dst_shift,), SENT_F, device=DEV))
        assert torch.equal(flat[dst_shift + T * d:], torch.full((EXTRA,), SENT_F, device=DEV)), (cs, 'wrote past dst')
        if det:
            assert torch.equal(call(), got), (cs, 'deterministic mode: two runs differ')
        assert_kernels(cs, call, scatter_kernels(det, vec) if n else set())
    mode = 'det' if det else 'default'
    if n == 0:
        exact('scatter ' + mode, cs, 'dst', cpu(got), cpu(base))
        return
    label = 'scatter %s %s' % (mode, 'vec' if vec and not det else ('sorted' if det else 'scalar'))
    if det:
        exact(label, cs, 'dst', cpu(got), seq_scatter(cpu(base), cpu(src), index))
    ti = torch.from_numpy(index).to(DEV)
    ref = base.double().index_add(0, ti, src.double())
    S = base.double().abs().index_add(0, ti, src.double().abs())
    nt = torch.bincount(ti, minlength=T).double()[:, None]
    check_bound(label, cs, 'dst', got, ref, (nt + 1) * U * S)


def scatter_index(kind, n, T, seed):
    rng = np.random.default_rng(seed)
    if kind == 'random':
        return rng.integers(0, T, n)
    if kind == 'distinct':
        return rng.permutation(T)[:n]
    if kind == 'hub':                              # 10^5 rows to one target among a few thousand others
        idx = rng.integers(0, T, n)
        idx[rng.permutation(n)[:100000]] = T // 3
        return idx
    raise ValueError(kind)


for _det in (0, 1):
    _m = '-det' if _det else ''
    for _d in (4, 6, 200, 256, 257, 1200):
        @case('scatter-d%d%s' % (_d, _m))
        def _(cs, d=_d, det=_det):
            run_scatter(cs, scatter_index('random', 5000, 700, d), 700, d, bool(det), seed=d)

    @case('scatter-d200-dst-offset-1%s' % _m)
    def _(cs, det=_det):
        run_scatter(cs, scatter_index('random', 3000, 500, 1), 500, 200, bool(det), dst_shift=1)

    @case('scatter-hub-1e5%s' % _m)
    def _(cs, det=_det):
        idx = scatter_index('hub', 130000, 4000, 2)
        assert int(np.bincount(idx).max()) >= 100000
        run_scatter(cs, idx, 4000, 256, bool(det))

    @case('scatter-distinct%s' % _m)
    def _(cs, det=_det):
        idx = scatter_index('distinct', 2000, 2000, 3)
        assert len(np.unique(idx)) == len(idx)
        run_scatter(cs, idx, 2000, 200, bool(det))

    @case('scatter-one-row%s' % _m)
    def _(cs, det=_det):
        run_scatter(cs, [9], 10, 257, bool(det))

    @case('scatter-no-rows%s' % _m)
    def _(cs, det=_det):
        run_scatter(cs, [], 10, 200, bool(det))


# the GRU dropout backward's own scatter forms (ld = 4h, seq_s / seq_r through row_seq), deterministic mode
@case('scatter-gru-dropout-bwd-det')
def _(cs):
    gru_dropout(cs, check_bwd=True)


# ---- Philox4x32-10 and the dropout masks -------------------------------------------------------------------------------------
PHILOX_M0, PHILOX_M1 = 0xD2511F53, 0xCD9E8D57
PHILOX_W0, PHILOX_W1 = 0x9E3779B9, 0xBB67AE85


def philox4x32_10(ctr, key):
    """numpy Philox4x32-10: ctr uint64 [n, 4] or [n] of 32-bit words (as uint64), key (k0, k1) -> uint32 [n, 4]"""
    M = np.uint64(0xFFFFFFFF)
    c = [np.asarray(w, dtype=np.uint64) & M for w in ctr]
    k0, k1 = np.uint64(key[0]) & M, np.uint64(key[1]) & M
    for r in range(10):
        p0 = c[0] * np.uint64(PHILOX_M0)
        p1 = c[2] * np.uint64(PHILOX_M1)
        hi0, lo0 = p0 >> np.uint64(32), p0 & M
        hi1, lo1 = p1 >> np.uint64(32), p1 & M
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0, k1 = (k0 + np.uint64(PHILOX_W0)) & M, (k1 + np.uint64(PHILOX_W1)) & M
    return np.stack(c, axis=-1).astype(np.uint32)


def mask_ref(seed, offset, n, p):
    """the scale factors of elements [offset, offset + n): Philox(counter = idx >> 2, key = seed), word idx & 3"""
    idx = np.uint64(offset) + np.arange(n, dtype=np.uint64)
    ctr = idx >> np.uint64(2)
    zero = np.zeros(n, dtype=np.uint64)
    r = philox4x32_10((ctr & np.uint64(0xFFFFFFFF), ctr >> np.uint64(32), zero, zero), (seed & 0xFFFFFFFF, seed >> 32))
    w = r[np.arange(n), (idx & np.uint64(3)).astype(np.int64)]
    u = w.astype(np.float32) * np.float32(2.0 ** -32)
    keep = np.float32(1.0) / (np.float32(1.0) - np.float32(p))
    return np.where(u >= np.float32(p), keep, np.float32(0.0)).astype(np.float32)


def run_mask(cs, seed, offset, n, p):
    _lib, L, P = lib()
    out = torch.full((n + EXTRA,), SENT_F, device=DEV)
    call = lambda: _lib.check(L.renet_dropout_mask(seed, offset, n, p, P(out), _lib.stream()), 'dropout_mask')
    call()
    got = cpu(out)
    assert (got[n:] == SENT_F).all(), (cs, 'mask wrote past n')
    exact('dropout mask', cs, 'mask', got[:n], mask_ref(seed, offset, n, p))
    assert_kernels(cs, call, {'dropout_mask_kernel'})
    return got[:n]


for _off in (0, 1, 2, 3, 5):
    for _p in (0.0, 0.5, 0.9):
        @case('mask-off%d-p%g' % (_off, _p))
        def _(cs, off=_off, p=_p):
            got = run_mask(cs, 0x1234_5678_9ABC_DEF1, off, 4099, p)
            if p > 0:                              # both outcomes occur
                assert (got == 0).any() and (got > 0).any()


@case('mask-counter-high-word')
def _(cs):
    off = (1 << 34) - 6                            # counters 2^32 - 2 .. 2^32 + 7: the high word turns non-zero inside
    assert (off >> 2) < (1 << 32) <= ((off + 37) >> 2)
    run_mask(cs, 42, off, 37, 0.5)


@case('mask-gru-fwd-x4-x3')
def _(cs):
    gru_dropout(cs, check_bwd=False)


def gru_dropout(cs, check_bwd):
    """renet_gru_fwd_dropout's materialised X4d / X3d against the restated masks on the gathered inputs; with check_bwd the
    deterministic backward's d_ent / d_rel against its dX4 column blocks"""
    _lib, L, P = lib()
    h, T, num_e, num_r, NH, p, seed = 200, 7, 900, 60, 300, 0.5, 0x0DDBA11_5EED
    rng = np.random.default_rng(21)
    lens = np.sort(rng.integers(1, 11, 300))[::-1].copy()
    lens[:3] = 10
    Q, S, max_len = len(lens), int(lens.sum()), int(lens.max())
    bs = np.array([int((lens > t).sum()) for t in range(max_len)], dtype=np.int32)
    gen = torch.Generator(device=DEV).manual_seed(22)
    g = lambda *s, sc=1.0: torch.randn(*s, device=DEV, generator=gen) * sc
    H2, ent, rel, glob = g(NH, h, sc=0.5), g(num_e, h, sc=0.3), g(num_r, h, sc=0.3), g(T, h, sc=0.1)
    readout = i32(rng.integers(0, NH, S))[:S]
    row_glob = i32(rng.integers(0, T, S))[:S]
    seq_s_np = rng.integers(0, 16, Q)              # 16 entities, 12 relations: ~ 100 rows per target
    seq_r_np = rng.integers(0, 12, Q)
    seq_s, seq_r = i32(seq_s_np)[:Q], i32(seq_r_np)[:Q]
    row_seq_np = np.repeat(np.arange(Q), lens)
    row_seq = i32(row_seq_np)[:S]
    seq_len, seq_start = i32(lens)[:Q], i32(np.concatenate(([0], np.cumsum(lens)[:-1])))[:Q]
    sc = 1.0 / h ** 0.5
    W = [g(3 * h, 4 * h, sc=sc), g(3 * h, h, sc=sc), g(3 * h, sc=0.1), g(3 * h, sc=0.1),
         g(3 * h, 3 * h, sc=sc), g(3 * h, h, sc=sc), g(3 * h, sc=0.1), g(3 * h, sc=0.1)]
    hn4, hn3 = torch.empty(Q, h, device=DEV), torch.empty(Q, h, device=DEV)
    nbytes = int(L.renet_gru_dropout_workspace_bytes(S, Q, T, h))
    ws = torch.empty(nbytes // 4, device=DEV)
    hbs = bs.ctypes.data_as(_lib.ctypes.c_void_p)
    prev = L.renet_set_gemm_engine(1)
    L.renet_set_weight_generation(-1)
    try:
        _lib.check(L.renet_gru_fwd_dropout(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel), P(row_seq), P(seq_s), P(seq_r),
                                           P(seq_len), P(seq_start), hbs, max_len, *[P(t) for t in W], P(hn4), P(hn3), S, Q, T, h,
                                           p, seed, P(ws), nbytes, _lib.stream()), 'gru_fwd_dropout')
        torch.cuda.synchronize()
        if not check_bwd:
            # X4d, X3d, zrow are the last three blocks of the forward workspace (gru.cu's carve)
            a4 = lambda x: (x + 3) // 4 * 4
            end = nbytes // 4 - a4(S)
            X3d = cpu(ws[end - a4(S * 3 * h):end - a4(S * 3 * h) + S * 3 * h]).reshape(S, 3 * h)
            X4d = cpu(ws[end - a4(S * 3 * h) - a4(S * 4 * h):][:S * 4 * h]).reshape(S, 4 * h)
            parts = [cpu(H2)[cpu(readout)], cpu(ent)[seq_s_np[row_seq_np]], cpu(rel)[seq_r_np[row_seq_np]], cpu(glob)[cpu(row_glob)]]
            x4 = np.concatenate(parts, axis=1)
            x3 = np.concatenate((parts[0], parts[1], parts[3]), axis=1)
            m4 = mask_ref(seed, 0, S * 4 * h, p).reshape(S, 4 * h)
            m3 = mask_ref(seed, S * 4 * h, S * 3 * h, p).reshape(S, 3 * h)
            assert 0.4 < (m3 == 0).mean() < 0.6
            exact('dropout mask', cs, 'X4d', X4d, x4 * m4)
            exact('dropout mask', cs, 'X3d', X3d, x3 * m3)
            return
        bbytes = int(L.renet_gru_bwd_dropout_workspace_bytes(S, Q, T, h))
        bws = torch.empty(bbytes // 4, device=DEV)
        dhn4, dhn3 = g(Q, h), g(Q, h)
        base_e, base_r = g(num_e, h, sc=0.1), g(num_r, h, sc=0.1)
        acc = {k: torch.randn_like(t) for k, t in (('dg', glob), ('w0', W[0]), ('w1', W[1]), ('w2', W[2]), ('w3', W[3]),
                                                   ('w4', W[4]), ('w5', W[5]), ('w6', W[6]), ('w7', W[7]))}

        def call():
            d_ent, d_rel, dH2 = base_e.clone(), base_r.clone(), torch.empty(NH, h, device=DEV)
            _lib.check(L.renet_gru_bwd_dropout(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel), P(row_seq), P(seq_s),
                                               P(seq_r), P(seq_len), P(seq_start), hbs, max_len, P(W[0]), P(W[1]), P(W[4]), P(W[5]),
                                               P(dhn4), P(dhn3), P(dH2), P(d_ent), P(d_rel), P(acc['dg']),
                                               *[P(acc['w%d' % k]) for k in range(8)], NH, S, Q, T, h, p, seed, P(ws), P(bws),
                                               bbytes, _lib.stream()), 'gru_bwd_dropout')
            return d_ent, d_rel

        with deterministic(True):
            d_ent, d_rel = call()
            torch.cuda.synchronize()
            a4 = lambda x: (x + 3) // 4 * 4
            start = bbytes // 4 - a4(S * 3 * h) - a4(S * 4 * h)   # dX4, dX3: the last two blocks (gru.cu's carve_bwd)
            dX4 = cpu(bws[start:start + S * 4 * h]).reshape(S, 4 * h)
            again = call()
            assert torch.equal(again[0], d_ent) and torch.equal(again[1], d_rel), (cs, 'deterministic mode: two runs differ')
            need = {'dropout_grad_rows_kernel', 'scatter_keys_kernel', 'cub', 'scatter_add_rows_sorted_kernel'}
            seen = kernels_of(call, need)
        assert need <= seen, sorted(seen)
        assert 'unpack_inputs_dropout_kernel' not in seen and 'scatter_add_rows_kernel' not in seen, sorted(seen)
    finally:
        L.renet_set_gemm_engine(prev)
    assert np.isfinite(dX4).all() and (dX4 != 0).mean() > 0.3
    for what, got, base, blk, key in (('d_ent', d_ent, base_e, 1, seq_s_np[row_seq_np]),
                                       ('d_rel', d_rel, base_r, 2, seq_r_np[row_seq_np])):
        src = np.ascontiguousarray(dX4[:, blk * h:(blk + 1) * h])
        assert np.bincount(key).max() >= 60
        exact('gru dropout bwd scatter det', cs, what, cpu(got), seq_scatter(cpu(base), src, key))
        ti = torch.from_numpy(key).to(DEV)
        s = torch.from_numpy(src).to(DEV).double()
        ref = base.double().index_add(0, ti, s)
        S_ = base.double().abs().index_add(0, ti, s.abs())
        nt = torch.bincount(ti, minlength=base.shape[0]).double()[:, None]
        check_bound('gru dropout bwd scatter fp64', cs, what, got, ref, (nt + 1) * U * S_)


# ---- renet_segment_pool_fwd / _bwd -------------------------------------------------------------------------------------------
def pool_ref(H, seg, mode):
    G, d = len(seg) - 1, H.shape[1]
    out = np.zeros((G, d), dtype=np.float32)
    arg = np.zeros((G, d), dtype=np.int64)
    for gi in range(G):
        r0, r1 = int(seg[gi]), int(seg[gi + 1])
        if r1 == r0:
            continue
        if mode == 1:
            out[gi] = H[r0:r1].max(0)
            arg[gi] = r0 + H[r0:r1].argmax(0)     # first maximum
        else:
            out[gi] = np.cumsum(H[r0:r1], axis=0, dtype=np.float32)[-1] / np.float32(r1 - r0)
    return out, arg


def run_pool(cs, lens, d, values='randn', seed=0):
    _lib, L, P = lib()
    rng = np.random.default_rng(seed)
    lens = np.asarray(lens, dtype=np.int64)
    seg = np.concatenate(([0], np.cumsum(lens)))
    N, G = int(seg[-1]), len(lens)
    if values == 'ties':
        H = rng.integers(-2, 3, (N, d)).astype(np.float32)
    elif values == 'negative':
        H = -np.abs(rng.standard_normal((N, d)).astype(np.float32)) - np.float32(1.0)
    else:
        H = rng.standard_normal((N, d)).astype(np.float32)
    if values == 'ninf':                           # segment 1 is all -inf; segment 2 has -inf in some columns only
        H[seg[1]:seg[2]] = -np.inf
        H[seg[2]:seg[3], ::3] = -np.inf
    Ht = torch.from_numpy(H).to(DEV)
    sp = i32(seg)[:G + 1]
    dout = torch.from_numpy(rng.standard_normal((G, d)).astype(np.float32)).to(DEV)
    for mode in (1, 0):
        mname = 'max' if mode else 'mean'
        out = torch.full((G * d + EXTRA,), SENT_F, device=DEV)
        arg = i32(np.zeros(0), G * d + EXTRA)
        call = lambda: _lib.check(L.renet_segment_pool_fwd(P(Ht), P(sp), G, d, mode, P(out), P(arg) if mode else None,
                                                           _lib.stream()), 'segment_pool_fwd')
        call()
        ref, rarg = pool_ref(H, seg, mode)
        got = cpu(out)
        assert (got[G * d:] == SENT_F).all(), (cs, 'fwd wrote past G*d')
        exact('pool %s fwd' % mname, cs, 'out', got[:G * d].reshape(G, d), ref)
        if mode:
            ga = cpu(arg)
            assert (ga[G * d:] == SENT_I).all()
            live = lens > 0
            exact('pool max argmax', cs, 'argmax', ga[:G * d].reshape(G, d)[live], rarg[live])
        assert_kernels(cs, call, {'segment_pool_fwd_kernel<%s>' % ('true' if mode else 'false')})
        dH = torch.full((N * d + EXTRA,), float('nan'), device=DEV)
        bcall = lambda: _lib.check(L.renet_segment_pool_bwd(P(dout), P(sp), P(arg) if mode else None, G, N, d, mode, P(dH),
                                                            _lib.stream()), 'segment_pool_bwd')
        bcall()
        exp = np.zeros((N, d), dtype=np.float32)
        dn = cpu(dout)
        for gi in range(G):
            r0, r1 = int(seg[gi]), int(seg[gi + 1])
            if r1 == r0:
                continue
            if mode:
                exp[rarg[gi], np.arange(d)] = dn[gi]
            else:
                exp[r0:r1] = dn[gi] / np.float32(r1 - r0)
        gd = cpu(dH)
        assert np.isnan(gd[N * d:]).all(), (cs, 'bwd wrote past N*d')
        exact('pool %s bwd' % mname, cs, 'dH', gd[:N * d].reshape(N, d), exp)
        if mode:
            assert (exp == 0).any(), 'rows outside every argmax exist'
        assert_kernels(cs, bcall, {'segment_max_bwd_kernel' if mode else 'segment_mean_bwd_kernel'})
    return H, seg


POOL_LENS = [0, 1, 5, 0, 0, 37, 1, 300, 2, 0]     # empty first, in a run in the middle and last; single rows
for _d in (1, 127, 128, 129, 200):
    @case('pool-d%d' % _d)
    def _(cs, d=_d):
        run_pool(cs, POOL_LENS, d, seed=d)

    @case('pool-ties-d%d' % _d)
    def _(cs, d=_d):
        run_pool(cs, POOL_LENS, d, 'ties', seed=d + 1)


@case('pool-1e5-row-segment')
def _(cs):
    run_pool(cs, [3, 100000, 0, 7], 129, seed=3)


@case('pool-all-negative')
def _(cs):
    run_pool(cs, POOL_LENS, 200, 'negative', seed=4)


@case('pool-all-ninf-segment')
def _(cs):
    H, seg = run_pool(cs, [4, 6, 9, 3], 130, 'ninf', seed=5)
    assert np.isneginf(H[seg[1]:seg[2]]).all()


# ---- renet_selfloop_gemm_bwd -------------------------------------------------------------------------------------------------
def selfloop_kernels(N, d_in, d_out, indexed, det, engine):
    """(fixed kernel names, whether the nn product runs on the packed tensor-core kernels)"""
    fixed = {'transpose_kernel'}
    umma = engine == 1 and d_out % 4 == 0 and d_in % 8 == 0 and N >= 64
    if not umma:
        fixed.add('sgemm_nn_kernel<false>' if d_out % 4 == 0 and d_in % 4 == 0 else 'sgemm_nn_naive')
    ix = 'true' if indexed else 'false'
    if d_in % 4 == 0 and d_out % 4 == 0:
        fixed |= {'sgemm_tn_splitk_kernel<%s,true>' % ix, 'sum_partials_kernel'} if det else {'sgemm_tn_splitk_kernel<%s,false>' % ix}
    else:
        fixed.add('sgemm_tn_naive')
    return fixed, umma


def run_selfloop(cs, N, d_in, d_out, indexed, det, hub=False, seed=0):
    _lib, L, P = lib()
    gen = torch.Generator(device=DEV).manual_seed(seed)
    rows = 23033 if indexed else N
    H = torch.randn(rows, d_in, device=DEV, generator=gen)
    h_index = None
    if indexed:
        h_index = torch.randint(0, rows, (N,), device=DEV, generator=gen, dtype=torch.int32)
        if hub:                                    # a third of the rows repeat 5 hub entities
            few = torch.randint(0, 5, (N,), device=DEV, generator=gen, dtype=torch.int32)
            h_index = torch.where(torch.rand(N, device=DEV, generator=gen) < 0.33, few, h_index)
    Wl = torch.randn(d_in, d_out, device=DEV, generator=gen) * 0.1
    dLoop = torch.randn(N, d_out, device=DEV, generator=gen)
    base = torch.randn(d_in, d_out, device=DEV, generator=gen) * 0.1
    ws = torch.empty(d_in * d_out, device=DEV)
    dH_buf = torch.empty(N * d_in + EXTRA, device=DEV)
    dW_buf = torch.empty(d_in * d_out + EXTRA, device=DEV)
    dH, dW = dH_buf[:N * d_in].view(N, d_in), dW_buf[:d_in * d_out].view(d_in, d_out)

    def call():
        dH_buf.fill_(float('nan'))
        dH_buf[N * d_in:] = SENT_F
        dW_buf[d_in * d_out:] = SENT_F
        dW.copy_(base)
        _lib.check(L.renet_selfloop_gemm_bwd(P(H), P(h_index), P(Wl), P(dLoop), P(dH), P(dW), P(ws), N, d_in, d_out, _lib.stream()),
                   'selfloop_gemm_bwd')
        return dH.clone(), dW.clone()

    engine = int(L.renet_get_gemm_engine())
    with deterministic(det):
        gH, gW = call()
        assert (cpu(dH_buf[N * d_in:]) == SENT_F).all() and (cpu(dW_buf[d_in * d_out:]) == SENT_F).all(), (cs, 'wrote past')
        if det:
            assert torch.equal(call()[1], gW), (cs, 'deterministic mode: dWloop differs across runs')
        fixed, umma = selfloop_kernels(N, d_in, d_out, indexed, det, engine)
        tc = {'umma_pack_b_kernel', 'umma_gemm_packed_kernel<false>', 'umma_gemm_resident_kernel<false>'}
        complete = lambda k: fixed <= k and (not umma or ('umma_pack_b_kernel' in k and len(k & tc) == 2))
        seen = kernels_of(call, complete)
        extra = seen - fixed
        ok = complete(seen) and (extra <= tc and len(extra) == 2 if umma else not extra)
        assert ok, '%s: ran %s, expected %s%s' % (cs, sorted(seen), sorted(fixed), ' + the packed GEMM' if umma else '')
    Hr = H[h_index.long()] if indexed else H
    ref = dLoop.double() @ Wl.double().t()
    S = dLoop.double().abs() @ Wl.double().abs().t()
    mode = ' det' if det else ''
    check_bound('selfloop dH', cs, 'dH', gH, ref, (d_out + 4) * U * S)
    refW = base.double() + Hr.double().t() @ dLoop.double()
    SW = base.double().abs() + Hr.double().abs().t() @ dLoop.double().abs()
    check_bound('selfloop dWloop' + mode, cs, 'dWloop', gW, refW, (N + 4) * U * SW)


for _det in (0, 1):
    _m = '-det' if _det else ''
    for _din, _dout in ((200, 200), (33, 100), (100, 33), (200, 100), (100, 200), (33, 33)):
        for _N in (1, 63, 1000):
            @case('selfloop-%dx%d-n%d%s' % (_din, _dout, _N, _m))
            def _(cs, din=_din, dout=_dout, N=_N, det=_det):
                run_selfloop(cs, N, din, dout, indexed=N > 1, det=bool(det), seed=N)

    @case('selfloop-layer1-34k-hubs%s' % _m)
    def _(cs, det=_det):
        run_selfloop(cs, 34000, 200, 200, indexed=True, det=bool(det), hub=True, seed=7)


# ---- renet_build_csr ---------------------------------------------------------------------------------------------------------
def key_bits(N):
    b = 1
    while (1 << b) < N and b < 31:
        b += 1
    return b


def run_csr(cs, dst, N, with_type=True, with_perm=True, seed=0):
    _lib, L, P = lib()
    rng = np.random.default_rng(seed)
    dst = np.asarray(dst, dtype=np.int64)
    E = len(dst)
    src = rng.integers(0, max(N, 1), E)
    et = rng.integers(0, 460, E)
    wsb = int(L.renet_csr_workspace_bytes(N, E))
    ws = torch.empty(max(wsb, 256), dtype=torch.uint8, device=DEV)
    outs = {k: i32(np.zeros(0), n + EXTRA) for k, n in (('row_ptr', N + 1), ('col_src', E), ('col_type', E), ('perm', E))}
    ins = [i32(a, 1) for a in (dst, src, et)]

    def call():
        for t in outs.values():
            t.fill_(SENT_I)
        _lib.check(L.renet_build_csr(P(ins[0]), P(ins[1]), P(ins[2]) if with_type else None, N, E, P(outs['row_ptr']),
                                     P(outs['col_src']) if E else None, P(outs['col_type']) if with_type and E else None,
                                     P(outs['perm']) if with_perm and E else None, P(ws), wsb, _lib.stream()),
                   'build_csr')

    call()
    order = np.argsort(dst, kind='stable')
    ref = {'row_ptr': np.concatenate(([0], np.cumsum(np.bincount(dst, minlength=N)))) if E else np.zeros(N + 1),
           'col_src': src[order], 'col_type': et[order], 'perm': order}
    for k, n in (('row_ptr', N + 1), ('col_src', E), ('col_type', E), ('perm', E)):
        got = cpu(outs[k])
        written = k in ('row_ptr', 'col_src') or (k == 'col_type' and with_type) or (k == 'perm' and with_perm)
        if written:
            exact('build_csr', cs, k, got[:n], ref[k].astype(np.int32))
            exact('build_csr', cs, k + ' sentinels', got[n:], np.full(EXTRA, SENT_I, dtype=np.int32))
        else:
            exact('build_csr', cs, k + ' untouched', got, np.full(n + EXTRA, SENT_I, dtype=np.int32))
    assert_kernels(cs, call, {'iota_kernel', 'cub', 'csr_finish_kernel'} if E else set())


for _N in (1, 2, 3, 4, 5, 65536, 65537):
    @case('csr-n%d' % _N)
    def _(cs, N=_N):
        rng = np.random.default_rng(N)
        E = 3 * N + 50
        dst = rng.integers(0, N, E)
        dst[:3] = N - 1                            # keys at N - 1, whose top bit is the highest sorted bit
        dst[-1] = N - 1
        b = key_bits(N)
        assert N - 1 < (1 << b) and (b == 1 or (1 << (b - 1)) < N), 'key_bits(N) is the fewest bits that hold N - 1'
        if N in (65536, 65537):
            assert b == {65536: 16, 65537: 17}[N] and (N - 1) >> (b - 1) == 1
        run_csr(cs, dst, N, seed=N)


@case('csr-one-key')
def _(cs):
    run_csr(cs, np.full(5000, 17), 40)


@case('csr-e0')
def _(cs):
    run_csr(cs, [], 33)


@case('csr-null-etype-perm')
def _(cs):
    run_csr(cs, np.random.default_rng(9).integers(0, 1000, 7000), 1000, with_type=False, with_perm=False)


# ---- renet_readout_subgraph --------------------------------------------------------------------------------------------------
def run_readout(cs, N, readout, seed=0):
    _lib, L, P = lib()
    rng = np.random.default_rng(seed)
    readout = np.asarray(readout, dtype=np.int64)
    S = len(readout)
    deg = rng.integers(0, 6, N)
    deg[readout[::3]] = 0                          # read-out nodes without in-edges
    rp = np.concatenate(([0], np.cumsum(deg)))
    E = int(rp[-1])
    col_src, col_type = rng.integers(0, N, E), rng.integers(0, 460, E)
    norm = (1.0 / np.maximum(deg, 1)).astype(np.float32) * rng.uniform(0.5, 1.5, N).astype(np.float32)
    ins = [i32(readout, 1), i32(rp, 1), i32(col_src, 1), i32(col_type, 1),
           torch.from_numpy(norm).to(DEV)]
    wsb = int(L.renet_readout_subgraph_workspace_bytes(N, S))
    ws = torch.empty(wsb // 4 + 1, dtype=torch.int32, device=DEV)
    sizes = {'uniq': S, 'readout_c': S, 'row_ptr2': S + 1, 'col_src2': E, 'col_type2': E, 'counts': 2}
    outs = {k: i32(np.zeros(0), n + EXTRA) for k, n in sizes.items()}
    norm2 = torch.full((S + EXTRA,), SENT_F, device=DEV)

    def call():
        ws.fill_(-99)                              # a dirty workspace: nothing may rely on it being zero
        for t in outs.values():
            t.fill_(SENT_I)
        norm2.fill_(SENT_F)
        o = outs
        _lib.check(L.renet_readout_subgraph(P(ins[0]), S, N, P(ins[1]), P(ins[2]), P(ins[3]), P(ins[4]), P(o['uniq']), P(o['readout_c']),
                                            P(o['row_ptr2']), P(o['col_src2']), P(o['col_type2']), P(norm2), P(o['counts']), P(ws),
                                            wsb, _lib.stream()), 'readout_subgraph')

    call()
    uq = np.unique(readout)
    Uc = len(uq)
    deg2 = np.zeros(S, dtype=np.int64)
    deg2[:Uc] = deg[uq]
    E2 = int(deg2.sum())
    ref = {'uniq': np.concatenate((uq, np.zeros(S - Uc, dtype=np.int64))), 'readout_c': np.searchsorted(uq, readout),
           'row_ptr2': np.concatenate(([0], np.cumsum(deg2))),
           'col_src2': np.concatenate([col_src[rp[v]:rp[v + 1]] for v in uq] + [np.zeros(0, np.int64)]),
           'col_type2': np.concatenate([col_type[rp[v]:rp[v + 1]] for v in uq] + [np.zeros(0, np.int64)]),
           'counts': np.array([Uc, E2])}
    valid = dict(sizes, col_src2=E2, col_type2=E2)
    for k, n in valid.items():
        got = cpu(outs[k])
        exact('readout_subgraph', cs, k, got[:n], ref[k].astype(np.int32))
        exact('readout_subgraph', cs, k + ' sentinels', got[n:], np.full(len(got) - n, SENT_I, dtype=np.int32))
    rn = np.concatenate((norm[uq], np.ones(S - Uc, dtype=np.float32)))
    gn = cpu(norm2)
    exact('readout_subgraph', cs, 'norm2', gn[:S], rn)
    exact('readout_subgraph', cs, 'norm2 sentinels', gn[S:], np.full(EXTRA, SENT_F, dtype=np.float32))
    assert_kernels(cs, call, {'rs_mark_kernel', 'cub', 'rs_compact_kernel', 'rs_copy_edges_kernel'})
    return Uc


@case('readout-duplicates')
def _(cs):
    rng = np.random.default_rng(1)
    ro = rng.integers(0, 5000, 3000)
    ro[7] = 4999                                   # node N - 1
    assert run_readout(cs, 5000, ro, 1) < 3000      # an unused capacity tail


@case('readout-all-distinct')
def _(cs):
    ro = np.random.default_rng(2).permutation(5000)[:2500]
    assert run_readout(cs, 5000, ro, 2) == 2500


@case('readout-one-node-repeated')
def _(cs):
    assert run_readout(cs, 300, np.full(700, 299), 3) == 1


@case('readout-s-greater-than-n')
def _(cs):
    ro = np.random.default_rng(4).integers(0, 50, 400)
    assert len(ro) > 50 and run_readout(cs, 50, ro, 4) <= 50


@case('readout-s1')
def _(cs):
    assert run_readout(cs, 10, [0], 5) == 1


# ---- renet_induce_edges ------------------------------------------------------------------------------------------------------
INDUCE_CHUNK = 1024


def graph_store(edge_counts, n_nodes, seed):
    """T graphs: graph t has n_nodes[t] local rows and edge_counts[t] edges sorted by local destination"""
    rng = np.random.default_rng(seed)
    srcs, dsts = [], []
    for E, n in zip(edge_counts, n_nodes):
        d = np.sort(rng.integers(0, n, E))
        srcs.append(rng.integers(0, n, E))
        dsts.append(d)
    off = np.concatenate(([0], np.cumsum(edge_counts))).astype(np.int64)
    Et = int(off[-1])
    return (off, np.concatenate(srcs + [np.zeros(0, np.int64)]), np.concatenate(dsts + [np.zeros(0, np.int64)]),
            rng.integers(0, 460, Et), rng.integers(0, 460, Et))


def run_induce(cs, store, n_nodes, comp_graph, keep, seed=0):
    """keep: per component, the probability that a local row is selected, or 'no-dst': the rows that are no edge's
    destination in that graph (so the component keeps no edge)"""
    _lib, L, P = lib()
    rng = np.random.default_rng(seed)
    off, gs, gd, ts, to = store
    G = len(comp_graph)
    mark_off = np.concatenate(([0], np.cumsum([n_nodes[g] for g in comp_graph])))
    cnt = np.array([off[g + 1] - off[g] for g in comp_graph], dtype=np.int64)
    cand_off = np.concatenate(([0], np.cumsum(cnt)))
    e_cand = int(cand_off[-1])
    newid = np.full(int(mark_off[-1]), -1, dtype=np.int64)
    nxt = 0
    for c, g in enumerate(comp_graph):            # batched ids ascend with (component, local row)
        if keep[c] == 'no-dst':
            sel = np.setdiff1d(np.arange(n_nodes[g]), gd[off[g]:off[g + 1]])
        else:
            sel = np.flatnonzero(rng.random(n_nodes[g]) < keep[c])
        newid[mark_off[c] + sel] = nxt + np.arange(len(sel))
        nxt += len(sel)
    N = nxt
    # reference: candidates in component order, survivors in candidate order
    ge = np.concatenate([off[g] + np.arange(off[g + 1] - off[g]) for g in comp_graph] + [np.zeros(0, np.int64)])
    comp_of = np.repeat(np.arange(G), cnt)
    s = newid[mark_off[comp_of] + gs[ge]] if e_cand else np.zeros(0, np.int64)
    d = newid[mark_off[comp_of] + gd[ge]] if e_cand else np.zeros(0, np.int64)
    live = (s >= 0) & (d >= 0)
    E = int(live.sum())
    rdst = d[live]
    assert np.all(np.diff(rdst) >= 0)
    deg = np.bincount(rdst, minlength=N)
    ref = {'row_ptr': np.concatenate(([0], np.cumsum(deg))), 'col_src': s[live], 'col_type_s': ts[ge][live],
           'col_type_o': to[ge][live], 'e_count': np.array([E])}
    ins = [torch.from_numpy(off).to(DEV)] + [i32(a, 1) for a in (gs, gd, ts, to, comp_graph, mark_off, cand_off, newid)]
    wsb = int(L.renet_induce_workspace_bytes(e_cand))
    ws = torch.empty(wsb // 4 + 1, dtype=torch.int32, device=DEV)
    sizes = {'row_ptr': N + 1, 'col_src': e_cand, 'col_type_s': e_cand, 'col_type_o': e_cand, 'e_count': 1}
    outs = {k: i32(np.zeros(0), n + EXTRA) for k, n in sizes.items()}
    norm = torch.full((N + EXTRA,), SENT_F, device=DEV)

    def call():
        ws.fill_(0)
        for t in outs.values():
            t.fill_(SENT_I)
        norm.fill_(SENT_F)
        o = outs
        _lib.check(L.renet_induce_edges(*[P(t) for t in ins], G, N, e_cand, P(o['row_ptr']), P(o['col_src']), P(o['col_type_s']),
                                        P(o['col_type_o']), P(norm), P(o['e_count']), P(ws), wsb, _lib.stream()), 'induce_edges')

    call()
    valid = dict(sizes, col_src=E, col_type_s=E, col_type_o=E)
    for k, n in valid.items():
        got = cpu(outs[k])
        exact('induce_edges', cs, k, got[:n], ref[k].astype(np.int32))
        exact('induce_edges', cs, k + ' sentinels', got[n:], np.full(len(got) - n, SENT_I, dtype=np.int32))
    rn = np.float32(1.0) / np.maximum(deg, 1).astype(np.float32)
    gn = cpu(norm)
    exact('induce_edges', cs, 'norm', gn[:N], rn)
    exact('induce_edges', cs, 'norm sentinels', gn[N:], np.full(EXTRA, SENT_F, dtype=np.float32))
    nblk = -(-e_cand // INDUCE_CHUNK)
    assert_kernels(cs, call, {'induce_scan_kernel', 'induce_rowptr_kernel'} | ({'induce_norm_kernel'} if N else set()) |
                   ({'induce_count_kernel', 'induce_emit_kernel'} if nblk else set()))
    return e_cand, nblk, E


@case('induce-carry-over-1024-blocks')
def _(cs):
    counts, nodes = [0, 420000, 0, 380000, 300000, 0], [50, 6000, 40, 5000, 4000, 30]
    store = graph_store(counts, nodes, 1)
    comp = [0, 1, 2, 3, 3, 4, 5]                   # empty components first, in the middle and last; two on graph 3
    e_cand, nblk, E = run_induce(cs, store, nodes, comp, [0.9, 0.9, 0.9, 0.9, 0.6, 0.9, 0.9], 1)
    assert e_cand > 1048576 and nblk > 1024, 'more than 1 048 576 candidates: the scan carries across 1024-block rounds'
    assert 0 < E < e_cand


@case('induce-empty-components')
def _(cs):
    counts, nodes = [0, 3000, 0, 0, 2500, 0], [10, 800, 5, 7, 700, 3]
    store = graph_store(counts, nodes, 2)
    comp = [0, 2, 1, 3, 2, 4, 5, 5]
    run_induce(cs, store, nodes, comp, [0.8] * len(comp), 2)


@case('induce-two-components-one-graph')
def _(cs):
    counts, nodes = [4000, 2000], [900, 500]
    store = graph_store(counts, nodes, 3)
    run_induce(cs, store, nodes, [0, 1, 0], [0.7, 0.9, 0.5], 3)


@case('induce-keeps-no-edge')
def _(cs):
    counts, nodes = [3000, 2000], [900, 500]
    store = graph_store(counts, nodes, 4)
    e_cand, nblk, E = run_induce(cs, store, nodes, [0, 1], ['no-dst', 'no-dst'], 4)
    assert E == 0 and e_cand == 5000 and nblk == 5


def summary():
    return ['%-30s worst %.3f  (%s %s)' % ((k,) + WORST[k]) for k in sorted(WORST)]
