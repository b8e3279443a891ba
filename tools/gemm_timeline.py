"""Where the packed 3xTF32 GEMM's time goes (run on the GPU box): per-warpgroup records through renet_debug_gemm_timing.

    python tools/gemm_timeline.py [M [indexed|plain]]      (default: the layer-1 self-loop, 34 500 rows through an index)

Prints, per warpgroup role, the median and maximum of the time spent waiting on operand barriers, in wgmma.wait_group, in
the epilogue and in the hi/lo split of A (resident kernel), and the work items per warpgroup."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from renet_b200 import _lib  # noqa: E402

M = int(sys.argv[1]) if len(sys.argv) > 1 else 34500
indexed = (sys.argv[2] if len(sys.argv) > 2 else 'indexed') == 'indexed'
N = K = 200
dev = torch.device('cuda:0')
L, P = _lib.lib(), _lib.ptr
_lib.ensure_scratch(dev)
L.renet_set_gemm_engine(1)
torch.manual_seed(0)
rows = 23033 if indexed else M
A = torch.randn(rows, K, device=dev) * 0.3
B = torch.randn(K, N, device=dev) * 0.1
idx = torch.randint(0, rows, (M,), device=dev, dtype=torch.int32) if indexed else None
out = torch.empty(M, N, device=dev)
SMS, SLOTS = 132, 4
buf = torch.zeros(SMS * SLOTS * 8, dtype=torch.int64, device=dev)
stream = _lib.stream()


def call():
    _lib.check(L.renet_selfloop_gemm(P(A), P(idx), P(B), P(out), M, K, N, stream), 'renet_selfloop_gemm')


for _ in range(5):
    call()
torch.cuda.synchronize()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
ev[0].record()
for _ in range(50):
    call()
ev[1].record()
torch.cuda.synchronize()
print('M %d N %d K %d %s: %.1f us per call (packing launch included), 50 calls' % (
    M, N, K, 'indexed' if indexed else 'plain', ev[0].elapsed_time(ev[1]) * 1e3 / 50))
L.renet_debug_gemm_timing(P(buf))
call()
torch.cuda.synchronize()
L.renet_debug_gemm_timing(None)
d = buf.cpu().numpy().reshape(SMS * SLOTS, 8)
d = d[d[:, 0] != 0].astype(np.float64)
role = (d[:, 7].astype(np.int64) >> 32)
items = (d[:, 7].astype(np.int64) & 0xffffffff)
clk = 1.98e3          # SM cycles per us at the maximum SM clock (clocks.max.sm 1980 MHz)
g0 = d[:, 0].min()
print('GEMM kernel span by the global timer: %.1f us (first entry -> last exit); entry skew max %.1f us' % (
    (d[:, 1].max() - g0) / 1e3, (d[:, 0].max() - g0) / 1e3))
ex = (d[:, 1] - g0) / 1e3
print('warpgroup exit after the first entry: min %.1f median %.1f max %.1f us' % (ex.min(), np.median(ex), ex.max()))
names = {0: 'streaming producer', 1: 'streaming consumer', 2: 'resident consumer'}
bars = {0: 'wait empty', 1: 'wait full', 2: 'wait B chunk'}
for r in sorted(set(role.tolist())):
    m = role == r
    print('%s (%d warpgroups), items per warpgroup min %d median %d max %d' % (
        names.get(r, r), m.sum(), items[m].min(), np.median(items[m]), items[m].max()))
    cols = [('span', d[m, 2]), (bars.get(r, 'barrier'), d[m, 3]), ('wgmma wait', d[m, 4]), ('epilogue', d[m, 5]),
            ('A split', d[m, 6])]
    for name, x in cols:
        if not x.any():
            continue
        x = x / clk
        print('  %-13s median %6.1f  max %6.1f us  (%4.1f %% of the median span)' % (
            name, np.median(x), x.max(), 100 * np.median(x) / max(np.median(d[m, 2] / clk), 1e-9)))
