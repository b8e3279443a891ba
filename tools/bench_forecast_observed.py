"""Forecasting over observed history (RENet.forecast_observed) on the synthetic ICEWS18-shaped split of
tools/bench_observed.py, on one GPU.  Prints one JSON line.

    python tools/bench_forecast_observed.py [--timestamps 40] [--test 4] [--valid 4] [--loop-queries 200] [--reps 3]

Every quadruple of the stream is a known fact; the queries are the test triples' (entity, relation, timestamp) rows in
both directions, each with its history window built from the facts by synthetic.observed_history (timed too, on the
host).  graph_dict and global_emb are bench_observed's (the true graphs; RENet_global.get_global_emb on the kernels).

  (a) forecast_observed over the queries of the first test timestamp and over the whole split, objects and subjects,
      k = 10 and 100, without a filter and with ``known`` = every quadruple as triples (the static filter; its
      FilterIndex is built inside each call): wall time ending in a device synchronise;
  (b) the per-query loop it replaces, over the first --loop-queries queries of the split (objects): _encode_one over the
      query's history, ``linear``, softmax, the known answers masked, torch.topk; ms per query and extrapolated.
(a) and (b) alternate --reps times after one warm-up of each.  The card's name and power limit are read in the same run."""
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

from bench_eval import DEV, H, gpu_info                                    # noqa: E402
from bench_observed import setup                                           # noqa: E402
from renet_b200 import synthetic                                           # noqa: E402
from renet_b200.inference import FilterIndex                               # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--timestamps', type=int, default=40)
    ap.add_argument('--valid', type=int, default=4)
    ap.add_argument('--test', type=int, default=4)
    ap.add_argument('--loop-queries', type=int, default=200)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_forecast_observed.py measures on a GPU; none is visible')
    name, power = gpu_info()
    quads, num_e, num_r, times, te, gd, ge, m, gm, split = setup(args.timestamps, args.valid, args.test)
    q = split[0]
    first = np.flatnonzero(q[:, 3] == q[0, 3])
    res = {'device': name, 'power_limit_w': power, 'h': H, 'num_e': num_e, 'num_r': num_r, 'known_facts': len(quads),
           'split_queries': len(q), 'timestamp_queries': len(first)}

    queries, history = {}, {}
    t0 = time.perf_counter()
    for subject, c in ((True, 0), (False, 2)):
        queries[subject] = np.stack((q[:, c], q[:, 1], q[:, 3]), 1)
        history[subject] = synthetic.observed_history(quads, q[:, c], q[:, 3], subject)
    res['observed_history_both_directions_ms'] = round((time.perf_counter() - t0) * 1e3, 1)

    def sub(subject, rows):
        hl, ht = history[subject]
        return queries[subject][rows], ([hl[i] for i in rows], [ht[i] for i in rows])

    scopes = {'timestamp': first, 'split': np.arange(len(q))}
    inputs = {(s, scope): sub(s, rows) for s in (True, False) for scope, rows in scopes.items()}
    configs = [(scope, s, k, kn) for scope in scopes for s in (True, False) for k in (10, 100) for kn in (False, True)]

    def forecast_ms(scope, subject, k, known):
        qq, hh = inputs[(subject, scope)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.forecast_observed(qq, hh, gd, ge, k=k, subject=subject, known=quads[:, :3] if known else None)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    fi = FilterIndex(quads)
    n_loop = min(args.loop_queries, len(q))

    def loop_ms():
        R = m.num_rels
        hl, ht = history[True]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad():
            for i, (e, r, _) in enumerate(queries[True][:n_loop]):
                s_h = torch.zeros(H, device=DEV) if len(hl[i]) == 0 else m._encode_one(int(e), int(r), hl[i], ht[i], True,
                                                                                       gd, ge)
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
    for _ in range(args.reps):
        for c in configs:
            fc[c].append(forecast_ms(*c))
        loops.append(loop_ms())
    for (scope, s, k, kn), v in fc.items():
        key = 'forecast_observed_%s_%s_k%d_%s_ms' % (scope, 'objects' if s else 'subjects', k, 'known' if kn else 'raw')
        res[key] = round(float(np.median(v)), 1)
        res[key + '_min_max'] = [round(float(min(v)), 1), round(float(max(v)), 1)]
    res['loop_queries_timed'] = n_loop
    res['loop_ms_per_query'] = round(float(np.median(loops)), 3)
    res['loop_ms_per_query_min_max'] = [round(float(min(loops)), 3), round(float(max(loops)), 3)]
    res['loop_extrapolated_split_s'] = round(res['loop_ms_per_query'] * len(q) / 1e3, 2)
    res['loop_extrapolated_timestamp_s'] = round(res['loop_ms_per_query'] * len(first) / 1e3, 2)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
