"""The relation head over observed history (RENet.evaluate_relations_observed) against the entity head's
evaluate_observed on the same synthetic ICEWS18-shaped split, on one GPU.  Prints one JSON line.

    python tools/bench_relations.py [--timestamps 40] [--test 4] [--valid 4] [--reps 5]

The split, histories, graphs and global embeddings are tools/bench_observed.py's.  Both calls run time-aware (raw,
filtered and time-aware ranks), alternating --reps times after one warm-up of each; each time is a host clock around the
call ending in a device synchronise, and CUDA events split the relation call into its encoding (_encode_queries) and its
ranking (_rank_rows).  Also reported: forecast_relations_observed's time for every test triple's subject (k = 10, known
relations left out time-aware), the distinct sequences each call encodes -- one per (entity, history) for the relation
head, one per (entity, relation, history) for the entity head -- and the relation MRRs.  The card's name and power limit
are read in the same run."""
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

from bench_eval import gpu_info                      # noqa: E402
from bench_observed import counts, setup             # noqa: E402
from renet_b200 import synthetic                     # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--timestamps', type=int, default=40)
    ap.add_argument('--valid', type=int, default=4)
    ap.add_argument('--test', type=int, default=4)
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_relations needs a GPU'
    name, power = gpu_info()
    quads, num_e, num_r, times, te, gd, ge, m, gm, split = setup(args.timestamps, args.valid, args.test)
    q, sh, oh = split
    n = len(q)
    res = {'gpu': name, 'power_limit_w': power, 'num_e': num_e, 'num_r': num_r, 'test_triples': n,
           'test_timestamps': args.test}
    c = counts(m, split, gd, ge)
    res['entity_head_sequences'] = c['subject_distinct_queries'] + c['object_distinct_queries']
    res['relation_head_sequences'] = 0
    for col, hist, nm in ((0, sh, 's_history'), (2, oh, 'o_history')):
        (_, _, hid, _), has = m._observed_histories(q[:, col], hist, nm, gd, ge)
        res['relation_head_sequences'] += int(len(np.unique(hid[has])))

    events = {'encode': [], 'rank': []}

    def evented(method, key):
        fn = getattr(m, method)

        def wrapper(*a, **kw):
            b, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            b.record()
            out = fn(*a, **kw)
            e.record()
            events[key].append((b, e))
            return out
        setattr(m, method, wrapper)
        return fn

    def timed(call, split_events=False):
        if split_events:
            orig = (evented('_encode_queries', 'encode'), evented('_rank_rows', 'rank'))
            for v in events.values():
                v.clear()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = call()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        if split_events:
            m._encode_queries, m._rank_rows = orig
            return ms, out, {k: sum(b.elapsed_time(e) for b, e in v) for k, v in events.items()}
        return ms, out

    rel = lambda: m.evaluate_relations_observed(q, sh, oh, gd, ge, total_data=quads, time_aware=True)   # noqa: E731
    ent = lambda: m.evaluate_observed(q, sh, oh, gd, ge, total_data=quads, time_aware=True)             # noqa: E731
    fq = np.stack((q[:, 0], q[:, 3]), 1)
    fh = synthetic.observed_history(quads, q[:, 0], q[:, 3], True)
    fc = lambda: m.forecast_relations_observed(fq, fh, gd, ge, k=10, known=quads, time_aware=True)    # noqa: E731
    timed(rel)                                           # warm-up: modules, GEMM packing, filter-index shapes
    timed(ent)
    timed(fc)
    tab = {'relations_observed_ms': [], 'relations_encode_ms': [], 'relations_rank_ms': [], 'entity_observed_ms': [],
           'forecast_relations_observed_ms': []}
    mrr = None
    for _ in range(args.reps):
        ms, out, ev = timed(rel, split_events=True)
        tab['relations_observed_ms'].append(ms)
        tab['relations_encode_ms'].append(ev['encode'])
        tab['relations_rank_ms'].append(ev['rank'])
        mrr = {k: out['protocols'][k]['mrr'] for k in out['protocols']}
        tab['entity_observed_ms'].append(timed(ent)[0])
        tab['forecast_relations_observed_ms'].append(timed(fc)[0])
    for k, v in tab.items():
        res[k] = round(float(np.median(v)), 3)
        res[k + '_min_max'] = [round(float(min(v)), 3), round(float(max(v)), 3)]
    res['relation_mrr'] = mrr
    print(json.dumps(res))


if __name__ == '__main__':
    main()
