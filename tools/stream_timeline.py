"""Where the stream gather kernel's time goes (run on the GPU box): per-warp time stamps through renet_debug_stream_timing.

    python tools/stream_timeline.py [icews18|gdelt] [hot]      ('hot' = pass the dataset's relation ranking)"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault('RENET_GATHER_KERNEL', 'stream')
from renet_b200 import _lib, hoststore, synthetic  # noqa: E402

preset = sys.argv[1] if len(sys.argv) > 1 else 'icews18'
use_hot = 'hot' in sys.argv[2:]
layer2 = 'layer2' in sys.argv[2:]          # non-indexed input rows (H [N,200]) instead of the embedding table through node_ent
dev = torch.device('cuda:0')
L, P = _lib.lib(), _lib.ptr
T = {'icews18': 240, 'gdelt': 2138, 'icews14': 181}[preset]
tkg = synthetic.SyntheticTKG(preset, seed=999, num_timestamps=T)
CTAS, MAX_WARPS = 132, 32      # the grid is one CTA per SM; no configuration runs more than 32 warps (StCfg)
R2 = 2 * tkg.num_r
gs = hoststore.GraphStore(tkg.graph_dict)
hs = hoststore.HistoryStore(tkg.s_hist, tkg.s_hist_t, tkg.quads[:, 0], gs)
hb = hoststore.assemble_view(hs.select(tkg.batch_indices(0, 1024, tail_only=False)), dev, device_edges=False)
g = hb.graph
torch.manual_seed(0)
ent = torch.randn(tkg.num_e, 200, device=dev) * 0.1
W = torch.randn(R2, 400, device=dev) * 0.1
out = torch.zeros(g.N, 200, device=dev)
Hrand = torch.randn(g.N, 200, device=dev)
Xin, xidx = (Hrand, None) if layer2 else (ent, g.node_ent)
hot = None
if use_hot:
    freq = np.zeros(R2, dtype=np.int64)
    for gg in tkg.graph_dict.values():
        freq += np.bincount(np.asarray(gg.type_s, dtype=np.int64), minlength=R2)
    hot = torch.from_numpy(np.argsort(-freq, kind='stable')[:128].astype(np.int32)).to(dev)
# room for the largest configuration: the kernel writes CTAS x (its warps) records of 8 stamps, packed from the start
buf = torch.zeros(CTAS * MAX_WARPS * 8, dtype=torch.int64, device=dev)
stream = _lib.stream()


def call():
    if hot is None:
        rc = L.renet_rgcn_gather(P(Xin), P(xidx), P(W), P(g.row_ptr), P(g.col_src), P(g.col_type_s), P(g.norm), P(out),
                                 g.N, g.E, 200, 200, 100, R2, 1, 1, stream)
    else:
        rc = L.renet_rgcn_gather_hot(P(Xin), P(xidx), P(W), P(g.row_ptr), P(g.col_src), P(g.col_type_s), P(g.norm), P(out),
                                     g.N, g.E, 200, 200, 100, R2, 1, 1, P(hot), hot.numel(), stream)
    _lib.check(rc, 'gather')


for _ in range(5):
    call()
torch.cuda.synchronize()
L.renet_debug_stream_timing(P(buf))
call()
torch.cuda.synchronize()
L.renet_debug_stream_timing(None)
rec = buf.cpu().numpy().reshape(-1, 8)
n_rec = int(np.count_nonzero(rec[:, 5]))         # every warp stamps its entry time: records written = CTAs x warps
assert n_rec % CTAS == 0 and not rec[n_rec:].any(), 'unexpected stamp layout (%d records)' % n_rec
WARPS = n_rec // CTAS
d = rec[:n_rec].reshape(CTAS, WARPS, 8).astype(np.float64)
clk = 1.98e3           # cycles per us at the maximum SM clock (H100 SXM: clocks.max.sm 1980 MHz)
g0 = d[:, :, 5].min()
print('N %d E %d; kernel span by the global timer: %.1f us (first entry -> last exit)' % (g.N, g.E, (d[:, :, 6].max() - g0) / 1e3))
print('CTA entry skew: max %.1f us; CTA exit (last warp) - global start: min %.1f / median %.1f / max %.1f us' % (
    (d[:, :, 5].min(1).max() - g0) / 1e3, (d[:, :, 6].max(1).min() - g0) / 1e3, np.median(d[:, :, 6].max(1) - g0) / 1e3,
    (d[:, :, 6].max(1).max() - g0) / 1e3))
part, pro, loop, tail = (d[:, :, 1] - d[:, :, 0]) / clk, (d[:, :, 2] - d[:, :, 1]) / clk, (d[:, :, 3] - d[:, :, 2]) / clk, (d[:, :, 4] - d[:, :, 3]) / clk
for name, x in (('partition search', part), ('rest of the prologue', pro), ('edge loop', loop), ('tail (hand-over, exit)', tail)):
    print('%-24s per warp: min %6.1f  median %6.1f  p90 %6.1f  max %6.1f us' % (name, x.min(), np.median(x), np.percentile(x, 90), x.max()))
n = d[:, :, 7]
print('edges per warp: min %d median %d max %d; per CTA: min %d median %d max %d' % (n.min(), np.median(n), n.max(), n.sum(1).min(), np.median(n.sum(1)), n.sum(1).max()))
per_edge = loop.sum() * clk / max(n.sum(), 1)
print('edge loop: %.0f SM cycles per edge per warp (%d warps share an SM: %.0f cycles per edge per SM)' % (per_edge, WARPS, per_edge / WARPS))
cta_loop = (d[:, :, 3].max(1) - d[:, :, 2].min(1)) / clk
print('per CTA first-edge -> last-edge: min %.1f median %.1f max %.1f us' % (cta_loop.min(), np.median(cta_loop), cta_loop.max()))
