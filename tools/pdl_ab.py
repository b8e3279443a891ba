"""Programmatic dependent launch, on and off in one process (DESIGN §5): bench.py's region-A step on the ICEWS18-shaped
workload, alternating RENET_PDL=0 / 1 per block of steps.  Prints, per mode, the GPU time per step (CUDA events around
the block) and the host time to enqueue one step (host clock around device_step, no synchronise, on an idle stream:
bursts of 4 steps after a synchronise, so a full launch queue never blocks the host), as one JSON line.

    python tools/pdl_ab.py [--steps 200] [--rounds 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from renet_b200 import _lib, hoststore, synthetic, utils  # noqa: E402
from renet_b200.model import RENet  # noqa: E402

H_DIM, NUM_BASES, BATCH = 200, 100, 1024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    tkg = synthetic.SyntheticTKG('icews18', seed=999, h_dim=H_DIM)
    torch.manual_seed(999)
    model = RENet(tkg.num_e, H_DIM, tkg.num_r, dropout=0).to(dev).eval()
    agg, ent, R2 = model.aggregator, model.ent_embeds.detach(), 2 * tkg.num_r
    W1, L1, W2, L2 = (agg.rgcn1.weight.detach(), agg.rgcn1.loop_weight.detach(), agg.rgcn2.weight.detach(),
                      agg.rgcn2.loop_weight.detach())
    hot_rel = hoststore.GraphStore(tkg.graph_dict).hot_relations(dev)
    pool = []
    for i in range(8):
        q, sh, oh = tkg.batch(i, BATCH, tail_only=False)
        dirs = []
        for hist, col, reverse in ((sh, 0, False), (oh, 2, True)):
            hb = utils.assemble_history_batch(hist[0], hist[1], q[:, col], tkg.graph_dict, dev)
            g = hb.graph
            dirs.append({'g': g, 'reverse': reverse, 'ct': g.col_type(reverse), 'sub': g.readout_sub(hb.readout, reverse),
                         'H1': torch.empty(g.N, H_DIM, device=dev), 'H2': torch.empty(hb.S, H_DIM, device=dev)})
        pool.append(dirs)
    L, P, stream = _lib.lib(), _lib.ptr, _lib.stream()
    step_no = [0]

    def device_step(dirs):
        step_no[0] += 1
        L.renet_set_weight_generation(step_no[0])
        for d in dirs:
            g, sub, hot = d['g'], d['sub'], hot_rel[d['reverse']]
            for H, idx, Wl, W, out, rows, rp, cs, ct, nm, ne, relu, hidx in (
                    (ent, g.node_ent, L1, W1, d['H1'], g.N, g.row_ptr, g.col_src, d['ct'], g.norm, g.E, 1, g.node_ent),
                    (d['H1'], sub.uniq, L2, W2, d['H2'], sub.N, sub.row_ptr, sub.col_src, sub.col_type(d['reverse']),
                     sub.norm, sub.E_cap, 0, None)):
                _lib.check(L.renet_selfloop_gemm(P(H), P(idx), P(Wl), P(out), rows, H_DIM, H_DIM, stream), 'gemm')
                _lib.check(L.renet_rgcn_gather_hot(P(H), P(hidx), P(W), P(rp), P(cs), P(ct), P(nm), P(out), rows, ne, H_DIM,
                                                   H_DIM, NUM_BASES, R2, relu, 1, P(hot), hot.numel(), stream), 'gather')
        L.renet_set_weight_generation(-1)

    for i in range(10):
        device_step(pool[i % len(pool)])
    torch.cuda.synchronize()
    res = {'0': {'ms_per_step': [], 'enqueue_us': []}, '1': {'ms_per_step': [], 'enqueue_us': []}}
    for r in range(args.rounds):
        for mode in ('0', '1'):
            os.environ['RENET_PDL'] = mode
            for i in range(5):
                device_step(pool[i % len(pool)])
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(args.steps):
                device_step(pool[i % len(pool)])
            b.record()
            torch.cuda.synchronize()
            host = []
            for i in range(args.steps):
                if i % 4 == 0:
                    torch.cuda.synchronize()
                t0 = time.perf_counter()
                device_step(pool[i % len(pool)])
                host.append(time.perf_counter() - t0)
            torch.cuda.synchronize()
            res[mode]['ms_per_step'].append(a.elapsed_time(b) / args.steps)
            res[mode]['enqueue_us'].append(float(np.median(host)) * 1e6)
    print(json.dumps({'device': torch.cuda.get_device_name(0), 'steps': args.steps, 'pdl_off': res['0'], 'pdl_on': res['1']}))


if __name__ == '__main__':
    main()
