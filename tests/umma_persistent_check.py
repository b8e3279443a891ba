"""Run in a subprocess by tests/test_gpu_umma_persistent.py: the persistent wgmma GEMM at the edges of its schedule.

The packed kernel splits M into 128-row x 104-column work units and hands each of at most 132 CTAs a contiguous range
of them.  The row counts below sit on and next to the unit and range boundaries; every output row must be written,
no row past M may be touched, and the error against fp64 stays within the 3xTF32 bar.  The decoder calls run the
fused cross-entropy epilogues (forward: partial logsumexp; backward: dlogits, then a split-K dX product)."""
import sys

import torch

sys.path.insert(0, __import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__))))
from renet_b200 import _lib  # noqa: E402
from renet_b200.decoder import decoder_cross_entropy  # noqa: E402

L = _lib.lib()
dev = 'cuda:0'
PAD = 64          # rows past M that must stay untouched
TOL = 2e-5

torch.manual_seed(0)
_lib.ensure_scratch(dev)          # the packed (persistent) kernel needs the scratch buffer for the packed B image
L.renet_set_gemm_engine(1)
worst = 0.0
for M in (64, 65, 64 * 132 - 1, 64 * 132, 64 * 132 + 1, 64 * 264 - 1, 64 * 264, 64 * 264 + 1, 2 * 64 * 132 + 1):
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

# decoder: EPI 1 (forward), EPI 2 and split-K dX (backward), against fp64; 23033 classes leave a 33-column last tile
for (M, N, K) in ((1024, 23033, 200), (300, 460, 200)):
    x = (torch.randn(M, K, device=dev) * 0.3).requires_grad_()
    W = (torch.randn(N, K, device=dev) * 0.05).requires_grad_()
    b = (torch.randn(N, device=dev) * 0.1).requires_grad_()
    tgt = torch.randint(0, N, (M,), device=dev)
    loss = decoder_cross_entropy(x, W, b, tgt)
    loss.backward()
    xd, Wd, bd = x.detach().double().requires_grad_(), W.detach().double().requires_grad_(), b.detach().double().requires_grad_()
    ref = torch.nn.functional.cross_entropy(xd @ Wd.t() + bd, tgt)
    ref.backward()
    e_loss = abs(loss.item() - ref.item()) / abs(ref.item())
    e_dx = (x.grad.double() - xd.grad).abs().max().item() / xd.grad.abs().max().item()
    e_dw = (W.grad.double() - Wd.grad).abs().max().item() / Wd.grad.abs().max().item()
    print('decoder M=%d N=%d K=%d rel err: loss %.2e dx %.2e dW %.2e' % (M, N, K, e_loss, e_dx, e_dw))
    assert e_loss < TOL and e_dx < 1e-4 and e_dw < 1e-4, (e_loss, e_dx, e_dw)
print('PERSISTENT_OK worst %.2e' % worst)
