"""Where the stream gather kernel's time goes (run on the GPU box): per-warp time stamps through renet_debug_stream_timing.

    python tools/stream_timeline.py [icews18|gdelt] [hot] [layer2|readout] [batch=1024]

'hot' = pass the dataset's relation ranking; 'layer2' = non-indexed input rows (H [N,200]) on the whole batched graph;
'readout' = layer 2 as the model runs it: the read-out sub-graph of the batch (renet_readout_subgraph: S compact
destinations, sources keep full-graph ids), launched with its edge capacity, linear, with the self-loop rows in the output.
RENET_GATHER_KERNEL picks the kernel (default here: stream); the time stamps need the stream kernel, the event-timed mean
(a rotation over four batches, stamps off) is printed for either."""
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
readout = 'readout' in sys.argv[2:]        # layer 2 on the read-out sub-graph
BATCH = int(([a[6:] for a in sys.argv[2:] if a.startswith('batch=')] or ['1024'])[0])
dev = torch.device('cuda:0')
L, P = _lib.lib(), _lib.ptr
T = {'icews18': 240, 'gdelt': 2138, 'icews14': 181}[preset]
tkg = synthetic.SyntheticTKG(preset, seed=999, num_timestamps=T)
CTAS, MAX_WARPS = 132, 32      # the grid is one CTA per SM; no configuration runs more than 32 warps (StCfg)
R2 = 2 * tkg.num_r
gs = hoststore.GraphStore(tkg.graph_dict)
hs = hoststore.HistoryStore(tkg.s_hist, tkg.s_hist_t, tkg.quads[:, 0], gs)
torch.manual_seed(0)
ent = torch.randn(tkg.num_e, 200, device=dev) * 0.1
W = torch.randn(R2, 400, device=dev) * 0.1
hot = None
if use_hot:
    freq = np.zeros(R2, dtype=np.int64)
    for gg in tkg.graph_dict.values():
        freq += np.bincount(np.asarray(gg.type_s, dtype=np.int64), minlength=R2)
    hot = torch.from_numpy(np.argsort(-freq, kind='stable')[:128].astype(np.int32)).to(dev)


def make_case(i):
    """launch arguments of one gather on batch i: (X, x_index, row_ptr, col_src, col_type, norm, out, N, E, relu, sizes)"""
    hb = hoststore.assemble_view(hs.select(tkg.batch_indices(i, BATCH, tail_only=False)), dev, device_edges=False)
    g = hb.graph
    Hrand = torch.randn(g.N, 200, device=dev)
    if readout:
        sub = g.readout_sub(hb.readout, False)
        U, E2 = sub.sizes()
        out = torch.randn(sub.N, 200, device=dev)      # stands in for the self-loop rows
        return (Hrand, None, sub.row_ptr, sub.col_src, sub.col_type(False), sub.norm, out, sub.N, sub.E_cap, 0,
                'S %d (U %d distinct) E2 %d (launched with E_cap %d), sources: %d rows' % (sub.N, U, E2, sub.E_cap, g.N))
    Xin, xidx = (Hrand, None) if layer2 else (ent, g.node_ent)
    return (Xin, xidx, g.row_ptr, g.col_src, g.col_type_s, g.norm, torch.zeros(g.N, 200, device=dev), g.N, g.E, 1,
            'N %d E %d' % (g.N, g.E))


cases = [make_case(i) for i in range(4)]
# room for the largest configuration: the kernel writes CTAS x (its warps) records of 8 stamps, packed from the start
buf = torch.zeros(CTAS * MAX_WARPS * 8, dtype=torch.int64, device=dev)
stream = _lib.stream()


def call(c):
    X, xi, rp, cs, ct, nm, out, N, E, relu, _ = c
    if hot is None:
        rc = L.renet_rgcn_gather(P(X), P(xi), P(W), P(rp), P(cs), P(ct), P(nm), P(out), N, E, 200, 200, 100, R2, relu, 1, stream)
    else:
        rc = L.renet_rgcn_gather_hot(P(X), P(xi), P(W), P(rp), P(cs), P(ct), P(nm), P(out), N, E, 200, 200, 100, R2, relu, 1,
                                     P(hot), hot.numel(), stream)
    _lib.check(rc, 'gather')


for _ in range(3):
    for c in cases:
        call(c)
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
reps = 25
ev[0].record()
for _ in range(reps):
    for c in cases:
        call(c)
ev[1].record()
torch.cuda.synchronize()
print('%s, kernel %s: mean %.1f us per launch (events, %d launches rotating over 4 batches, stamps off)' % (
    cases[0][-1], os.environ['RENET_GATHER_KERNEL'], ev[0].elapsed_time(ev[1]) * 1e3 / (reps * len(cases)), reps * len(cases)))
if os.environ['RENET_GATHER_KERNEL'][0] != 's':
    sys.exit(0)
L.renet_debug_stream_timing(P(buf))
call(cases[0])
torch.cuda.synchronize()
L.renet_debug_stream_timing(None)
rec = buf.cpu().numpy().reshape(-1, 8)
n_rec = int(np.count_nonzero(rec[:, 5]))         # every warp stamps its entry time: records written = CTAs x warps
assert n_rec % CTAS == 0 and not rec[n_rec:].any(), 'unexpected stamp layout (%d records)' % n_rec
WARPS = n_rec // CTAS
d = rec[:n_rec].reshape(CTAS, WARPS, 8).astype(np.float64)
clk = 1.98e3           # cycles per us at the maximum SM clock (H100 SXM: clocks.max.sm 1980 MHz)
g0 = d[:, :, 5].min()
print('one launch on batch 0, %d warps per CTA; kernel span by the global timer: %.1f us (first entry -> last exit)' % (
    WARPS, (d[:, :, 6].max() - g0) / 1e3))
print('CTA entry skew: max %.1f us; CTA exit (last warp) - global start: min %.1f / median %.1f / max %.1f us' % (
    (d[:, :, 5].min(1).max() - g0) / 1e3, (d[:, :, 6].max(1).min() - g0) / 1e3, np.median(d[:, :, 6].max(1) - g0) / 1e3,
    (d[:, :, 6].max(1).max() - g0) / 1e3))
part, pro, loop, tail = (d[:, :, 1] - d[:, :, 0]) / clk, (d[:, :, 2] - d[:, :, 1]) / clk, (d[:, :, 3] - d[:, :, 2]) / clk, (d[:, :, 4] - d[:, :, 3]) / clk
for name, x in (('partition search', part), ('rest of the prologue', pro), ('edge loop', loop), ('tail (hand-over, exit)', tail)):
    print('%-24s per warp: min %6.1f  median %6.1f  p90 %6.1f  max %6.1f us' % (name, x.min(), np.median(x), np.percentile(x, 90), x.max()))
first = (d[:, :, 2] - d[:, :, 0]) / clk
print('%-24s per warp: min %6.1f  median %6.1f  p90 %6.1f  max %6.1f us' % ('entry -> first edge', first.min(), np.median(first),
                                                                          np.percentile(first, 90), first.max()))
n = d[:, :, 7]
print('edges per warp: min %d median %d max %d; per CTA: min %d median %d max %d' % (n.min(), np.median(n), n.max(), n.sum(1).min(), np.median(n.sum(1)), n.sum(1).max()))
per_edge = loop.sum() * clk / max(n.sum(), 1)
print('edge loop: %.0f SM cycles per edge per warp (%d warps share an SM: %.0f cycles per edge per SM)' % (per_edge, WARPS, per_edge / WARPS))
cta_loop = (d[:, :, 3].max(1) - d[:, :, 2].min(1)) / clk
print('per CTA first-edge -> last-edge: min %.1f median %.1f max %.1f us' % (cta_loop.min(), np.median(cta_loop), cta_loop.max()))
