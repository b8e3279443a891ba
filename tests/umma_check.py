"""Run in a subprocess by tests/test_gpu_umma.py: wgmma 3xTF32 GEMM vs fp64 and vs the FFMA kernel."""
import sys

import numpy as np
import torch

sys.path.insert(0, __import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__))))
from renet_b200 import _lib  # noqa: E402

L = _lib.lib()
dev = 'cuda:0'


def gemm(A, idx, B, M):
    out = torch.full((M, B.shape[1]), float('nan'), device=dev)
    rc = L.renet_selfloop_gemm(_lib.ptr(A), _lib.ptr(idx), _lib.ptr(B), _lib.ptr(out), M, A.shape[1], B.shape[1], _lib.stream())
    _lib.check(rc, 'renet_selfloop_gemm')
    torch.cuda.synchronize()
    return out


torch.manual_seed(0)
worst = 0.0
for (M, N, K, indexed) in ((34483, 200, 200, True), (8573, 1200, 200, False), (962, 600, 200, False), (129, 200, 600, False),
                           (128, 200, 40, False), (5000, 408, 80, True)):
    rows = 23033 if indexed else M
    A = torch.randn(rows, K, device=dev) * 0.3
    B = torch.randn(K, N, device=dev) * 0.1
    idx = torch.randint(0, rows, (M,), device=dev, dtype=torch.int32) if indexed else None
    ref = (A[idx.long()] if indexed else A).double() @ B.double()
    L.renet_set_gemm_engine(0)
    ffma = gemm(A, idx, B, M)
    L.renet_set_gemm_engine(1)
    n0 = _lib.launch_count()
    umma = gemm(A, idx, B, M)
    scale = ref.abs().max().item()
    e_ffma = (ffma.double() - ref).abs().max().item() / scale
    e_umma = (umma.double() - ref).abs().max().item() / scale
    print('M=%d N=%d K=%d indexed=%s  rel err: ffma %.2e  umma(3xTF32) %.2e' % (M, N, K, indexed, e_ffma, e_umma))
    assert not torch.isnan(umma).any(), 'umma left outputs unwritten'
    assert e_umma < 2e-5, e_umma
    worst = max(worst, e_umma)
# timing at the self-loop shape
A = torch.randn(23033, 200, device=dev); B = torch.randn(200, 200, device=dev) * 0.1
idx = torch.randint(0, 23033, (34483,), device=dev, dtype=torch.int32)
for eng, name in ((0, 'ffma'), (1, 'umma')):
    L.renet_set_gemm_engine(eng)
    out = torch.empty(34483, 200, device=dev)
    for _ in range(3):
        L.renet_selfloop_gemm(_lib.ptr(A), _lib.ptr(idx), _lib.ptr(B), _lib.ptr(out), 34483, 200, 200, _lib.stream())
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(20):
        L.renet_selfloop_gemm(_lib.ptr(A), _lib.ptr(idx), _lib.ptr(B), _lib.ptr(out), 34483, 200, 200, _lib.stream())
    b.record(); torch.cuda.synchronize()
    print('selfloop GEMM 34483x200x200 %s: %.1f us' % (name, a.elapsed_time(b) / 20 * 1e3))
# engine 1 without scratch = v1 (self-staged B); with scratch = v2 (packed B + TMA)
L.renet_set_scratch(None, 0)
A = torch.randn(5000, 200, device=dev); B = torch.randn(200, 200, device=dev) * 0.1
ref = A.double() @ B.double()
L.renet_set_gemm_engine(1)
v1 = gemm(A, None, B, 5000)
e1 = (v1.double() - ref).abs().max().item() / ref.abs().max().item()
print('v1 (no scratch) rel err %.2e' % e1)
assert e1 < 2e-5
print('UMMA_OK worst %.2e' % worst)
