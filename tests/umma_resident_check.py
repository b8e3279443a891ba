"""Run in a subprocess by tests/test_gpu_umma_resident.py: the resident-panel wgmma GEMM at the edges of its schedule.

The self-loop product (N = K = 200) has two panels (104-column halves of the packed B); each gets half of the CTAs, and
a CTA's three warpgroups take its 64-row tiles in turn.  The row counts below sit on and next to the tile boundaries,
leave warpgroups without a tile (64, 65, 127) and give every CTA several (8 448, 34 500).  Every output row must be
written, no row past M may be touched, and the error against fp64 stays within the 3xTF32 bar."""
import sys

import torch

sys.path.insert(0, __import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__))))
from renet_b200 import _lib  # noqa: E402

L = _lib.lib()
dev = 'cuda:0'
PAD = 64          # rows past M that must stay untouched
TOL = 2e-5

torch.manual_seed(0)
_lib.ensure_scratch(dev)
L.renet_set_gemm_engine(1)
worst = 0.0
for M in (64, 65, 127, 128, 64 * 66 * 2, 64 * 66 * 2 + 1, 8448, 34500):
    for indexed in (False, True):
        N = K = 200
        rows = 23033 if indexed else M
        A = torch.randn(rows, K, device=dev) * 0.3
        B = torch.randn(K, N, device=dev) * 0.1
        idx = torch.randint(0, rows, (M,), device=dev, dtype=torch.int32) if indexed else None
        out = torch.full((M + PAD, N), float('nan'), device=dev)
        _lib.check(L.renet_selfloop_gemm(_lib.ptr(A), _lib.ptr(idx), _lib.ptr(B), _lib.ptr(out), M, K, N, _lib.stream()),
                   'renet_selfloop_gemm')
        torch.cuda.synchronize()
        ref = (A[idx.long()] if indexed else A).double() @ B.double()
        got = out[:M]
        assert not torch.isnan(got).any(), 'M=%d indexed=%s: outputs left unwritten' % (M, indexed)
        assert torch.isnan(out[M:]).all(), 'M=%d indexed=%s: rows past M were written' % (M, indexed)
        err = (got.double() - ref).abs().max().item() / ref.abs().max().item()
        print('M=%d indexed=%s rel err %.2e' % (M, indexed, err))
        assert err < TOL, err
        worst = max(worst, err)
print('RESIDENT_OK worst %.2e' % worst)
