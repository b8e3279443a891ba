"""Forecasting (RENet.forecast) on synthetic ICEWS18- and GDELT-shaped streams, set up as tools/bench_eval.py sets them up, on
one GPU.  Prints one JSON line.

    python tools/bench_forecast.py [--datasets icews18,gdelt] [--num-k 1000] [--loop-queries 200] [--reps 3]

  (a) forecast over the queries of the first test timestamp (latest_time is that timestamp, so no roll-over runs): ms per
      timestamp for both directions, k = 10 and 100, without and with the static filter of every known triple;
  (b) the per-query loop forecast replaces, over the first --loop-queries queries of that timestamp (objects of
      (s, r, ?)): _encode_one, ``linear``, softmax, the known answers masked, torch.topk; ms per query and extrapolated
      to the timestamp;
  (c) renet_decoder_topk with the filter's lists against renet_decoder_group_topk (R = 1, weight 1, ORDER_VALUE) on the
      same rows (one per query of the timestamp, seeded), timed with CUDA events: what the lists cost.
Every timed window ends in a device synchronise; (a) and (b) alternate --reps times after one warm-up of each."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from bench_eval import DEV, H, SeededGlobal, gpu_info, restore, setup, snapshot    # noqa: E402
from renet_b200.decoder import ORDER_VALUE, decoder_group_topk, decoder_topk      # noqa: E402
from renet_b200.inference import FilterIndex                                        # noqa: E402


def bench_dataset(ds, num_k, loop_queries, reps):
    tkg, m, te, _ = setup(ds, num_k, 3)
    quads = tkg.quads
    gm = SeededGlobal(tkg.num_e)
    snap = snapshot(m)
    first = te[quads[te, 3] == quads[te[0], 3]]
    q = quads[first]
    queries = {True: np.stack((q[:, 0], q[:, 1], q[:, 3]), 1), False: np.stack((q[:, 2], q[:, 1], q[:, 3]), 1)}
    out = {'num_e': tkg.num_e, 'num_r': tkg.num_r, 'num_k': num_k, 'queries_per_timestamp': len(first)}
    configs = [(subject, k, known) for subject in (True, False) for k in (10, 100) for known in (False, True)]

    def forecast_ms(subject, k, known):
        restore(m, snap)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.forecast(queries[subject], gm, k=k, subject=subject, known=quads if known else None)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    fi = FilterIndex(quads)
    n_loop = min(loop_queries, len(first))

    def loop_ms():
        restore(m, snap)
        R = m.num_rels
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad():
            for e, r, _ in queries[True][:n_loop]:
                hist, hist_t = m.s_hist_test[e], m.s_hist_test_t[e]
                s_h = torch.zeros(H, device=DEV) if len(hist) == 0 else m._encode_one(int(e), int(r), hist, hist_t, True)
                p = torch.softmax(m.linear(torch.cat((m.ent_embeds[int(e)], s_h, m.rel_embeds[:R][int(r)]))), dim=0)
                b, en = fi.ranges('objects', [e], [r])
                p[torch.from_numpy(fi.col('objects')[b[0]:en[0]].astype(np.int64)).to(DEV)] = -1.0
                torch.topk(p, 10)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / n_loop

    for c in configs:                                          # warm up every shape
        forecast_ms(*c)
    loop_ms()
    fc = {c: [] for c in configs}
    loops = []
    for _ in range(reps):
        for c in configs:
            fc[c].append(round(forecast_ms(*c), 1))
        loops.append(round(loop_ms(), 2))
    out['forecast_ms_per_timestamp'] = {'%s_k%d_%s' % ('objects' if s else 'subjects', k, 'filtered' if kn else 'raw'): v
                                        for (s, k, kn), v in fc.items()}
    out['loop_ms_per_query'] = loops
    out['loop_queries_timed'] = n_loop
    out['loop_ms_per_timestamp_extrapolated'] = [round(x * len(first), 0) for x in loops]

    # (c) the top-k kernels alone on one timestamp's rows
    rows = len(first)
    gen = torch.Generator().manual_seed(7)
    x = (torch.randn(rows, 3 * H, generator=gen) * 0.2).to(DEV)
    b_o, e_o = fi.ranges('objects', q[:, 0], q[:, 1])
    ex = tuple(torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(DEV) for a in (fi.col('objects'), b_o, e_o))
    w, b = m.linear.weight.detach(), m.linear.bias.detach()
    ones = torch.ones(rows, device=DEV)
    out['kernel_rows'] = rows
    out['kernel_list_len_mean'] = round(float(np.mean(e_o - b_o)), 2)
    calls = {'group_topk': lambda k: decoder_group_topk(x, w, b, ones, 1, k, ORDER_VALUE),
             'topk_no_lists': lambda k: decoder_topk(x, w, b, k),
             'topk_lists': lambda k: decoder_topk(x, w, b, k, ex)}
    with torch.no_grad():
        for k in (10, 100):
            for name, fn in calls.items():
                fn(k)
                times = []
                for _ in range(max(reps, 10)):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fn(k)
                    e1.record()
                    e1.synchronize()
                    times.append(round(e0.elapsed_time(e1), 3))
                out['kernel_ms_%s_k%d' % (name, k)] = times
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--datasets', default='icews18,gdelt')
    ap.add_argument('--num-k', type=int, default=1000)
    ap.add_argument('--loop-queries', type=int, default=200)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_forecast.py measures on a GPU; none is visible')
    name, power = gpu_info()
    res = {'device': name, 'power_limit_w': power, 'h': H}
    for ds in a.datasets.split(','):
        res[ds] = bench_dataset(ds, a.num_k, a.loop_queries, a.reps)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
