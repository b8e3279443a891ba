"""Run in a subprocess by tests/test_gpu_gemm_contract.py: every kernel of the dense-GEMM engine in every argument form the
library's callers use, against float64 on the same fp32 operands.

Each case goes through renet_debug_gemm, which runs one product exactly as the library dispatches it (or on a forced kernel)
and names the kernel that ran; the case asserts that name, so a dispatch change cannot move a case off the kernel it covers.
C is a flat buffer holding the written window -- rows < M, columns [n0, n0 + N) of ldc, for every batch entry -- inside
sentinels: NaN, or a random base when the case accumulates, in PAD rows past M, in every column of ldc outside the window and
between the windows of batch entries.  After the call the window must match the fp64 reference (base + A[idx] @ B + bias)
within the kernel's bar, measured as max-abs-diff / max-abs-ref, and every other element must be bitwise unchanged.

Where two kernels claim the same k order and product order for every output element (resident and streaming at K <= 224,
the deduplicated product and the resident one), the same operands are also run on the other kernel and must give a
bitwise-equal C.

The shapes are those of the callers:
  * the self-loop product (N = K = 200, indexed through node_ent, up to 34.5 k rows; at least 16 384 indexed rows deduplicate);
  * the GRU input projections (gru.cu launch_gru_fwd): GI / PQ / PT with ldc = 6h, the entity projection with the bias, the
    relation projection accumulating into a 3h-wide window, T or Q rows that can be fewer than 64, and the dropout / dense
    projections (K = 4h or 3h) into the column windows [0, 3h) and [3h, 6h);
  * the batched recurrent products: both encoders in one launch, entry b reading columns b*h of A and writing columns
    b*3h of C (forward step loop), or reading b*3h and accumulating into b*h (backward, every training step), with M = n_act
    down to 1;
  * the weight gradients (tn form): dW_loop over ~34 k indexed nodes, the GRU dW_hh reduction over (L - 1) * Q rows into the
    right half of dWhh, and the written (not accumulated) input-projection gradients;
  * the FFMA engine (renet_set_gemm_engine(0)), the FFMA fall-backs (N % 8 != 0, fewer than 64 rows, a pointer 4 bytes
    off 16-byte alignment);
  * two products with different B enqueued at once on two streams, each packing its B into its own stream's block."""
import collections
import ctypes
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from renet_b200 import _lib  # noqa: E402

L = _lib.lib()
dev = 'cuda:0'
PAD = 16            # sentinel rows past M
FFMA_TILED, FFMA_NAIVE, STREAMING, RESIDENT, DEDUP = 1, 2, 4, 5, 6
NAMES = {FFMA_TILED: 'ffma-tiled', FFMA_NAIVE: 'ffma-naive', STREAMING: 'streaming', RESIDENT: 'resident', DEDUP: 'dedup'}
FORMS = {'nn': 0, 'prepacked': 1, 'tn': 2}
TOL = {FFMA_TILED: 1e-5, FFMA_NAIVE: 1e-5, STREAMING: 2e-5, RESIDENT: 2e-5, DEDUP: 2e-5}
ENT_ROWS = 23033    # ICEWS18 entities: the table the indexed products gather from

stream = _lib.stream()
L.renet_set_weight_generation(-1)       # no packed-weight cache: every product packs its B


def addr(t, off=0):
    return ctypes.c_void_p(t.data_ptr() + 4 * off)


def packed_bytes(N, K):
    return -(-N // 200) * -(-K // 32) * 53248


count = collections.Counter()
forms_seen = collections.Counter()
worst = collections.defaultdict(float)
n_cases = 0


def case(name, expect, M, N, K, form='nn', kernel=0, engine=1, indexed=False, bias=False, acc=False, batch=1,
         lda=None, batch_a=None, a_off=0, ldb=None, b_off=0, ldc=None, batch_c=None, n0=0, same_as=()):
    """One product.  A, B and C are flat buffers; entry b of A / C starts batch_a / batch_c elements after entry 0 (the GRU's
    column-interleaved encoders), C's window starts at column n0 of ldc; a_off shifts A off its allocation (a_off = 1: 4
    bytes off 16-byte alignment).  same_as: forced kernels that must reproduce C bitwise on the same operands."""
    global n_cases
    torch.manual_seed(n_cases)
    n_cases += 1
    tn = form == 'tn'
    if tn:                               # C[M, N] (+)= A[idx]^T @ B: A is [K rows, M columns used], B [K, N]
        a_rows = ENT_ROWS if indexed else K
        a_cols = M
    else:
        a_rows = ENT_ROWS if indexed else M
        a_cols = K
    batch_a = a_cols if batch_a is None else batch_a
    lda = (batch - 1) * batch_a + a_cols if lda is None else lda
    ldb = N if ldb is None else ldb
    batch_c = N if batch_c is None else batch_c
    ldc = n0 + (batch - 1) * batch_c + N if ldc is None else ldc
    assert lda >= (batch - 1) * batch_a + a_cols and ldc >= n0 + (batch - 1) * batch_c + N
    scale_a = 0.3 if not tn else 0.05
    A = torch.randn(a_off + a_rows * lda, device=dev) * scale_a
    b_rows = K
    B = torch.randn(b_off + batch * b_rows * ldb, device=dev) * 0.1
    batch_b = b_rows * ldb
    n_idx = K if tn else M
    idx = torch.randint(0, a_rows, (n_idx,), device=dev, dtype=torch.int32) if indexed else None
    bvec = torch.randn(batch, N, device=dev) * 0.5 if bias else None
    c_rows = M + PAD
    C0 = torch.randn(c_rows * ldc, device=dev) if acc else torch.full((c_rows * ldc,), float('nan'), device=dev)

    # fp64 reference of the window, and the flat positions it covers
    ref = []
    pos = []
    cols = torch.arange(N, device=dev)
    rws = torch.arange(M, device=dev)
    for b in range(batch):
        Ab = torch.as_strided(A, (a_rows, a_cols), (lda, 1), a_off + b * batch_a).double()
        Bb = torch.as_strided(B, (b_rows, N), (ldb, 1), b_off + b * batch_b).double()
        if indexed:
            Ab = Ab[idx.long()]
        r = Ab.t() @ Bb if tn else Ab @ Bb
        if bias:
            r = r + bvec[b].double()
        p = (n0 + b * batch_c + rws[:, None] * ldc + cols[None, :]).reshape(-1)
        if acc:
            r = r + C0[p].double().view(M, N)
        ref.append(r.reshape(-1))
        pos.append(p)
    ref, pos = torch.cat(ref), torch.cat(pos)
    outside = torch.ones(c_rows * ldc, dtype=torch.bool, device=dev)
    outside[pos] = False
    assert pos.numel() == batch * M * N and int((~outside).sum()) == pos.numel(), 'windows overlap'

    ws_bytes = batch * packed_bytes(N, K)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)

    # C's window starts at column n0 of each row: C + n0 is the base pointer
    def run_at(kern):
        Cx = C0.clone()
        L.renet_set_gemm_engine(engine)
        try:
            got = L.renet_debug_gemm(FORMS[form], kern, addr(A, a_off), _lib.ptr(idx), lda, addr(B, b_off), ldb, addr(Cx, n0),
                                     ldc, _lib.ptr(bvec), M, N, K, int(acc), batch, batch_a, batch_b, batch_c, _lib.ptr(ws),
                                     ws_bytes, stream)
        finally:
            L.renet_set_gemm_engine(1)
        if got < 0:
            _lib.check(got, 'renet_debug_gemm(%s)' % name)
        torch.cuda.synchronize()
        return got, Cx

    got_kernel, Cx = run_at(kernel)
    assert got_kernel == expect, '%s: served by %s, expected %s' % (name, NAMES.get(got_kernel, got_kernel), NAMES[expect])
    w = Cx[pos].double()
    assert not torch.isnan(w).any(), '%s: outputs left unwritten' % name
    err = ((w - ref).abs().max() / ref.abs().max()).item()
    bad = outside & (Cx.view(torch.int32) != C0.view(torch.int32))
    if bad.any():
        first = int(bad.nonzero()[0])
        raise AssertionError('%s: %d sentinel(s) changed, first at row %d column %d (ldc %d)' % (
            name, int(bad.sum()), first // ldc, first % ldc, ldc))
    assert err < TOL[got_kernel], '%s (%s): error %.3e > %.0e' % (name, NAMES[got_kernel], err, TOL[got_kernel])
    line = '%-44s %-10s M=%-6d N=%-5d K=%-5d err %.2e' % (name, NAMES[got_kernel], M, N, K, err)
    for other in same_as:
        k2, C2 = run_at(other)
        assert k2 == other, '%s: forced %s, served by %s' % (name, NAMES[other], NAMES.get(k2, k2))
        assert torch.equal(C2.view(torch.int32), Cx.view(torch.int32)), '%s: %s differs from %s, max %.3e' % (
            name, NAMES[other], NAMES[got_kernel], (C2[pos] - Cx[pos]).abs().max().item())
        line += '  == %s' % NAMES[other]
        count[other] += 1
    print(line, flush=True)
    count[got_kernel] += 1
    forms_seen[(form, got_kernel)] += 1
    worst[got_kernel] = max(worst[got_kernel], err)


# ---- the self-loop product (N = K = 200): row counts on and next to the resident kernel's 64-row tiles and CTA ranges, the
#      streaming kernel's 128-row units and 132-CTA ranges (forced), the deduplication threshold, and the benchmark's sizes
for M in (64, 65, 127, 128, 64 * 132 - 1, 64 * 132, 64 * 132 + 1, 64 * 264 - 1, 64 * 264, 64 * 264 + 1, 8448, 34500):
    case('selfloop plain', RESIDENT, M, 200, 200, same_as=(STREAMING,))
for M in (64, 65, 127, 128, 64 * 132 - 1, 64 * 132, 64 * 132 + 1, 8448, 16383):
    case('selfloop indexed', RESIDENT, M, 200, 200, indexed=True, same_as=(STREAMING,))
for M in (16384, 64 * 264 - 1, 64 * 264, 64 * 264 + 1, 34483, 34500):
    case('selfloop indexed, deduplicated', DEDUP, M, 200, 200, indexed=True, same_as=(RESIDENT,))
case('selfloop deduplicated, bias, column window', DEDUP, 16384, 200, 200, indexed=True, bias=True, ldc=1200, n0=600,
     same_as=(RESIDENT,))
case('selfloop engine 0', FFMA_TILED, 34500, 200, 200, indexed=True, engine=0)
case('selfloop 5000 rows', RESIDENT, 5000, 200, 200)
case('selfloop indexed, 34483 rows', DEDUP, 34483, 200, 200, indexed=True, same_as=(RESIDENT,))
case('selfloop indexed, 8449 rows', RESIDENT, 8449, 200, 200, indexed=True)

# ---- K: partly filled last k-step (4, 12, 28), the resident maximum (224), the first streaming K (228), the GRU's 3h / 4h
for K in (4, 12, 28, 200, 224):
    case('K axis', RESIDENT, 1153, 200, K, same_as=(STREAMING,))
    case('K axis, engine 0', FFMA_TILED, 1153, 200, K, engine=0)
for K in (228, 600, 800):
    case('K axis', STREAMING, 1153, 200, K)
    case('K axis, engine 0', FFMA_TILED, 1153, 200, K, engine=0)
case('K axis, indexed, accumulate', STREAMING, 129, 200, 228, indexed=True, acc=True)
case('K = 40, N = 104', RESIDENT, 128, 104, 40, same_as=(STREAMING,))

# ---- N: one 8-column group, 104-column halves and their neighbours, the GRU's 3h / 6h, a non-multiple of 8
for N in (8, 96, 104, 112, 200, 208, 600, 1200):
    case('N axis', RESIDENT, 1153, N, 200, same_as=(STREAMING,))
    case('N axis, K = 228', STREAMING, 1153, N, 228)
for N in (104, 112, 208, 600):
    case('N axis, accumulate', RESIDENT, 1153, N, 200, acc=True, same_as=(STREAMING,))
case('N = 196 (N % 8 != 0)', FFMA_TILED, 1153, 196, 200)
case('N = 196, engine 0', FFMA_TILED, 1153, 196, 200, engine=0)
case('N = 196, accumulate, bias, window', FFMA_TILED, 129, 196, 200, acc=True, bias=True, ldc=208, n0=4)

# ---- fewer than 64 rows: the nn form leaves them to the FFMA engine, the prepacked form keeps them on the tensor cores
for M in (1, 7, 63):
    case('M < 64, nn', FFMA_TILED, M, 200, 200, indexed=True)
    case('M < 64, prepacked', RESIDENT, M, 200, 200, form='prepacked', indexed=True, same_as=(STREAMING,))
    case('M < 64, prepacked K = 800', STREAMING, M, 600, 800, form='prepacked', ldc=1200, n0=600)

# ---- earlier single-call checks of the engine (wgmma vs fp64 and FFMA), kept as inputs
for (M, N, K, ix, kern) in ((34483, 200, 200, True, DEDUP), (8573, 1200, 200, False, RESIDENT), (962, 600, 200, False, RESIDENT),
                            (129, 200, 600, False, STREAMING), (128, 200, 40, False, RESIDENT), (5000, 408, 80, True, RESIDENT)):
    case('engine check', kern, M, N, K, indexed=ix)
    case('engine check, engine 0', FFMA_TILED, M, N, K, indexed=ix, engine=0)

# ---- GRU input projections at h = 200 (prepacked, as gru.cu issues them): GI over the read-out rows, PQ with the bias
#      (entity part) then accumulating the relation part into columns [0, 3h), PT over the timestamps
for M in (1, 7, 63, 64, 65, 129, 1153, 3000):
    case('GRU PQ ent: indexed, bias, N = 6h', RESIDENT, M, 1200, 200, form='prepacked', indexed=True, bias=True,
         same_as=(STREAMING,))
    case('GRU PQ rel: indexed, accumulate, [0, 3h) of 6h', RESIDENT, M, 600, 200, form='prepacked', indexed=True, acc=True,
         ldc=1200, same_as=(STREAMING,))
for M in (1, 37):
    case('GRU PT: T rows', RESIDENT, M, 1200, 200, form='prepacked', same_as=(STREAMING,))
case('GRU GI: read-out rows', RESIDENT, 3000, 1200, 200, form='prepacked', indexed=True)
# ... at h = 400 the panels do not fit: the streaming kernel, the bias across 12 column tiles
case('GRU PQ ent h=400: bias, N = 6h', STREAMING, 1153, 2400, 400, form='prepacked', indexed=True, bias=True)
case('GRU PQ rel h=400: accumulate, [0, 3h)', STREAMING, 1153, 1200, 400, form='prepacked', indexed=True, acc=True, ldc=2400)
# ... h = 200 through the nn form (the FFMA engine's packed weights, and sgemm_nn under engine 1)
case('GRU PQ ent, nn, engine 0', FFMA_TILED, 1153, 1200, 200, indexed=True, bias=True, engine=0)
case('GRU PQ rel, nn, engine 0', FFMA_TILED, 1153, 600, 200, indexed=True, acc=True, ldc=1200, engine=0)
case('GRU PQ rel, nn', RESIDENT, 1153, 600, 200, indexed=True, acc=True, ldc=1200)
# ... dropout / dense inputs: X4 @ W_ih4^T into [0, 3h), X3 @ W_ih3^T into [3h, 6h)
for M in (1, 129, 3000):
    case('GRU dropout X4: K = 4h, [0, 3h) of 6h', STREAMING, M, 600, 800, form='prepacked', ldc=1200)
    case('GRU dropout X3: K = 3h, [3h, 6h) of 6h', STREAMING, M, 600, 600, form='prepacked', ldc=1200, n0=600)
case('GRU dense X4: K = h', RESIDENT, 1153, 600, 200, form='prepacked', ldc=1200, same_as=(STREAMING,))

# ---- batched recurrent products (two encoders per launch)
for M in (1, 7, 63, 64, 65, 127, 128, 129, 1153, 3000):
    # backward h = 200: dHprev[:, b*h:(b+1)*h] += dGH[:, b*3h:(b+1)*3h] @ W_hh_b
    case('GRU bwd: batch 2, accumulate, K = 3h', STREAMING, M, 200, 600, form='prepacked', batch=2, acc=True)
for M in (1, 129, 1153):
    # forward step loop h = 400 (the recurrence kernel declines h > 224): GH[:, b*3h:] = Hprev[:, b*h:] @ W_hh_b^T
    case('GRU fwd step h=400: batch 2', STREAMING, M, 1200, 400, form='prepacked', batch=2)
    # the same at h = 200: the resident kernel with one panel range per encoder
    case('GRU fwd step h=200: batch 2', RESIDENT, M, 600, 200, form='prepacked', batch=2, same_as=(STREAMING,))
    # backward h = 400
    case('GRU bwd h=400: batch 2, accumulate, K = 3h', STREAMING, M, 400, 1200, form='prepacked', batch=2, acc=True)
# a bias per batch entry, and sentinel columns between the entries' windows
case('batch 2, bias, gaps', RESIDENT, 1153, 200, 200, form='prepacked', batch=2, bias=True, acc=True, batch_c=208, n0=4,
     ldc=420, same_as=(STREAMING,))
case('batch 2, bias, gaps, K = 228', STREAMING, 1153, 200, 228, form='prepacked', batch=2, bias=True, acc=True, batch_c=208,
     n0=4, ldc=420, indexed=True)

# ---- lda > K, A 4 bytes off 16-byte alignment (FFMA naive), forced FFMA under engine 1
case('lda > K', RESIDENT, 1153, 200, 200, lda=212, indexed=True, same_as=(STREAMING,))
case('lda > K, engine 0', FFMA_TILED, 1153, 200, 200, lda=212, indexed=True, engine=0)
case('unaligned A', FFMA_NAIVE, 1153, 200, 200, a_off=1)
case('unaligned A, engine 0, bias, accumulate', FFMA_NAIVE, 129, 600, 200, a_off=1, engine=0, bias=True, acc=True, ldc=1200,
     n0=600)
case('forced FFMA naive', FFMA_NAIVE, 129, 208, 228, kernel=FFMA_NAIVE, indexed=True, acc=True)
case('forced FFMA tiled', FFMA_TILED, 1153, 1200, 200, kernel=FFMA_TILED, bias=True)
case('N = 6h, indexed, bias', RESIDENT, 1153, 1200, 200, indexed=True, bias=True)
case('K = 4h, bias, window', STREAMING, 1153, 600, 800, bias=True, ldc=1200, n0=600)

# ---- tn form (FFMA split-K): dW_loop, the GRU dW_hh reduction, the written input-projection gradients
case('tn dW_loop: indexed, accumulate', FFMA_TILED, 200, 200, 34500, form='tn', indexed=True, acc=True)
case('tn dW_loop: layer 2 rows', FFMA_TILED, 200, 200, 8449, form='tn', acc=True)
# dWhh[:, 3h:] += Hs[1:, h:2h]^T @ dGH[1:, 3h:6h] over (L - 1) * Q rows
case('tn GRU dW_hh: right half, accumulate', FFMA_TILED, 200, 600, 15 * 3000, form='tn', acc=True, lda=400, a_off=200,
     ldb=1200, b_off=600, ldc=1200, n0=600)
case('tn GRU dB_row: written, window', FFMA_TILED, 200, 600, 1153, form='tn', indexed=True, ldc=1208, n0=4)
case('tn unaligned', FFMA_NAIVE, 200, 600, 1153, form='tn', acc=True, a_off=1)
case('tn forced naive', FFMA_NAIVE, 100, 300, 2000, form='tn', kernel=FFMA_NAIVE, indexed=True)


def two_streams():
    """Two self-loop products with different B enqueued back to back on two non-blocking streams (torch's pool streams),
    with no synchronisation between them: each packs its B while the other's kernels may still read theirs.  Each must
    match fp64 and leave its sentinel rows untouched."""
    global n_cases
    torch.manual_seed(n_cases)
    n_cases += 1
    M, N, K = 34500, 200, 200
    runs = []
    for indexed, kern in ((True, DEDUP), (False, RESIDENT)):
        A = torch.randn(ENT_ROWS if indexed else M, K, device=dev) * 0.3
        B = torch.randn(K, N, device=dev) * 0.1
        idx = torch.randint(0, A.shape[0], (M,), device=dev, dtype=torch.int32) if indexed else None
        C0 = torch.full((M + PAD, N), float('nan'), device=dev)
        runs.append((kern, A, B, idx, C0, C0.clone(), torch.cuda.Stream(device=dev)))
    torch.cuda.synchronize()
    got = [L.renet_debug_gemm(FORMS['nn'], 0, _lib.ptr(A), _lib.ptr(idx), K, _lib.ptr(B), N, _lib.ptr(C), N, None, M, N, K,
                              0, 1, 0, 0, 0, None, 0, ctypes.c_void_p(s.cuda_stream))
           for kern, A, B, idx, C0, C, s in runs]
    torch.cuda.synchronize()
    for g, (kern, A, B, idx, C0, C, s) in zip(got, runs):
        if g < 0:
            _lib.check(g, 'renet_debug_gemm(two streams)')
        assert g == kern, 'two streams: served by %s, expected %s' % (NAMES.get(g, g), NAMES[kern])
        ref = (A[idx.long()] if idx is not None else A).double() @ B.double()
        assert not torch.isnan(C[:M]).any(), 'two streams (%s): outputs left unwritten' % NAMES[kern]
        err = ((C[:M].double() - ref).abs().max() / ref.abs().max()).item()
        assert torch.equal(C[M:].view(torch.int32), C0[M:].view(torch.int32)), 'two streams (%s): sentinels changed' % (
            NAMES[kern])
        assert err < TOL[kern], 'two streams (%s): error %.3e > %.0e' % (NAMES[kern], err, TOL[kern])
        print('%-44s %-10s M=%-6d N=%-5d K=%-5d err %.2e' % ('two streams', NAMES[kern], M, N, K, err), flush=True)
        count[kern] += 1
        worst[kern] = max(worst[kern], err)


two_streams()

print('cases per kernel: ' + ', '.join('%s %d' % (NAMES[k], count[k]) for k in sorted(count)))
print('forms: ' + ', '.join('%s/%s %d' % (f, NAMES[k], n) for (f, k), n in sorted(forms_seen.items())))
print('worst error per kernel: ' + ', '.join('%s %.2e' % (NAMES[k], worst[k]) for k in sorted(worst)))
assert set(count) == set(NAMES), 'a kernel was never reached: %s' % sorted(set(NAMES) - set(count))
print('GEMM_CONTRACT_OK %d cases' % n_cases)
