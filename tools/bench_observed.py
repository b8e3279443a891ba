"""Evaluation over observed history (RENet.evaluate_observed) on a synthetic ICEWS18-shaped split, on one GPU.  Prints one
JSON line.

    python tools/bench_observed.py [--timestamps 40] [--test 4] [--valid 4] [--loop-triples 200] [--reps 3]

synthetic.make_quads('icews18') is cut into train / valid / test by timestamp; the per-triple histories come from
synthetic.build_history over the whole stream, the graphs from build_graph_dict, and global_emb from RENet_global's
get_global_emb over every timestamp (both models on the kernels, deterministic parameters).

  (a) evaluate_observed over the whole test split, time_aware=True (raw, filtered and time-aware ranks) and raw only: wall
      time ending in a device synchronise, and CUDA events around the encoding (_encode_queries) and the ranking
      (_rank_triples) of the time-aware run; rows, distinct queries and distinct (entity, timestamp) components;
  (b) the per-triple loop it replaces, in host order over the first --loop-triples test triples: _encode_one for each
      direction, ``linear``, rank_with_ties and the filtered ranks; ms per triple and extrapolated to the split;
  (c) evaluate_stream_batched over the first two test timestamps (one roll-over, driven by the same global model): ms per
      timestamp, for comparison.
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

from bench_eval import DEV, H, gpu_info, restore, snapshot, timed_method    # noqa: E402
from renet_b200 import synthetic                                             # noqa: E402
from renet_b200.global_model import RENet_global                             # noqa: E402
from renet_b200.inference import _same_time, rank_with_ties                  # noqa: E402
from renet_b200.model import RENet                                           # noqa: E402


def setup(T, n_valid, n_test):
    quads, num_e, num_r = synthetic.make_quads('icews18', seed=11, num_timestamps=T)
    times = np.unique(quads[:, 3])
    t_valid, t_test = times[-(n_valid + n_test)], times[-n_test]
    tr = np.flatnonzero(quads[:, 3] < t_valid)
    te = np.flatnonzero(quads[:, 3] >= t_test)
    gd = synthetic.build_graph_dict(quads, num_r)
    S, ST, O, OT = synthetic.build_history(quads)
    torch.manual_seed(0)
    m = RENet(num_e, H, num_r, dropout=0, model=0, seq_len=10, num_k=1000).to(DEV).eval()
    gm = RENet_global(num_e, H, num_r, dropout=0, model=3, seq_len=10, num_k=1000, maxpool=1).to(DEV).eval()
    with torch.no_grad():
        ge = gm.get_global_emb([int(t) for t in times], gd)
    pick = lambda L, idx: [L[i] for i in idx]                                  # noqa: E731
    m.graph_dict = {int(t): gd[int(t)] for t in times if t < t_test}
    m.global_emb = {int(t): ge[int(t)] for t in times if t < t_test}
    m.init_history(quads[tr], (pick(S, tr), pick(ST, tr)), (pick(O, tr), pick(OT, tr)), [], ([], []), ([], []),
                   quads[te], (pick(S, te), pick(ST, te)), (pick(O, te), pick(OT, te)))
    m.latest_time = torch.tensor(int(t_test))            # as test.py starts: the first test timestamp rolls nothing
    split = (quads[te], (pick(S, te), pick(ST, te)), (pick(O, te), pick(OT, te)))
    return quads, num_e, num_r, times, te, gd, ge, m, gm, split


def counts(m, split, gd, ge):
    """Rows, distinct queries and distinct (entity, timestamp) components of each direction, as evaluate_observed plans
    them."""
    q, sh, oh = split
    out = {'rows': 2 * len(q)}
    for c, hist, name in ((0, sh, 's_history'), (2, oh, 'o_history')):
        (hl, ht, hid, ent_of), has = m._observed_histories(q[:, c], hist, name, gd, ge)
        keys = np.unique(hid[has] * m.num_rels + q[has, 1])
        hids = np.unique(hid[has])
        side = 'subject' if c == 0 else 'object'
        out['%s_distinct_queries' % side] = int(len(keys))
        out['%s_components' % side] = int(len({(int(ent_of[x]), int(t)) for x in hids for t in ht[x]}))
        out['%s_history_entries' % side] = int(sum(len(ht[x]) for x in hids))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--timestamps', type=int, default=40)
    ap.add_argument('--valid', type=int, default=4)
    ap.add_argument('--test', type=int, default=4)
    ap.add_argument('--loop-triples', type=int, default=200)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_observed needs a GPU'
    name, power = gpu_info()
    quads, num_e, num_r, times, te, gd, ge, m, gm, split = setup(args.timestamps, args.valid, args.test)
    q, sh, oh = split
    n = len(q)
    known = torch.from_numpy(quads).to(DEV)
    res = {'gpu': name, 'power_limit_w': power, 'num_e': num_e, 'num_r': num_r, 'test_triples': n,
           'test_timestamps': args.test}
    res.update(counts(m, split, gd, ge))

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

    def observed_ms(time_aware, split_events=False):
        if split_events:
            orig = (evented('_encode_queries', 'encode'), evented('_rank_triples', 'rank'))
            for v in events.values():
                v.clear()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = m.evaluate_observed(q, sh, oh, gd, ge, total_data=quads, time_aware=time_aware)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        if split_events:
            m._encode_queries, m._rank_triples = orig
            return ms, out, {k: sum(b.elapsed_time(e) for b, e in v) for k, v in events.items()}
        return ms, out

    n_loop = min(args.loop_triples, n)

    def loop_ms():
        R = m.num_rels
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad():
            for i in range(n_loop):
                trip = torch.from_numpy(q[i]).to(DEV)
                s, r, o = (int(x) for x in q[i, :3])
                s_h = torch.zeros(H, device=DEV) if len(sh[0][i]) == 0 else m._encode_one(s, r, sh[0][i], sh[1][i], True, gd, ge)
                o_h = torch.zeros(H, device=DEV) if len(oh[0][i]) == 0 else m._encode_one(o, r, oh[0][i], oh[1][i], False, gd, ge)
                ob = m.linear(torch.cat((m.ent_embeds[s], s_h, m.rel_embeds[:R][r])))
                sub = m.linear(torch.cat((m.ent_embeds[o], o_h, m.rel_embeds[R:][r])))
                rank_with_ties(sub, s), rank_with_ties(ob, o)
                m._filtered_ranks(trip, sub, ob, known)
                m._filtered_ranks(trip, sub, ob, _same_time(known, trip))
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    observed_ms(True)                                     # warm-up: modules, GEMM packing, filter-index shapes
    observed_ms(False)
    loop_ms()
    tab = {'observed_time_aware_ms': [], 'observed_raw_ms': [], 'encode_ms': [], 'rank_ms': [], 'loop_ms_per_triple': []}
    mrr = None
    for _ in range(args.reps):
        ms, out, ev = observed_ms(True, split_events=True)
        tab['observed_time_aware_ms'].append(ms)
        tab['encode_ms'].append(ev['encode'])
        tab['rank_ms'].append(ev['rank'])
        mrr = {k: out['protocols'][k]['mrr'] for k in out['protocols']}
        tab['observed_raw_ms'].append(observed_ms(False)[0])
        tab['loop_ms_per_triple'].append(loop_ms() / n_loop)
    for k, v in tab.items():
        res[k] = round(float(np.median(v)), 3)
        res[k + '_min_max'] = [round(float(min(v)), 3), round(float(max(v)), 3)]
    res['loop_triples'] = n_loop
    res['loop_extrapolated_split_s'] = round(res['loop_ms_per_triple'] * n / 1e3, 2)
    res['mrr'] = mrr

    # (c) evaluate_stream_batched over the first two test timestamps: one roll-over
    t_test = np.unique(q[:, 3])
    two = np.flatnonzero(q[:, 3] <= t_test[1])
    snap = snapshot(m)
    acc = {}
    timed_method(m, '_roll_over', acc)
    sub = (q[two], ([sh[0][i] for i in two], [sh[1][i] for i in two]), ([oh[0][i] for i in two], [oh[1][i] for i in two]))
    stream_ms = []
    for _ in range(2):                                     # first run warms the roll-over's shapes
        restore(m, snap)
        acc.clear()
        torch.manual_seed(5)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.evaluate_stream_batched(*sub, gm, total_data=quads, time_aware=True)
        torch.cuda.synchronize()
        stream_ms.append((time.perf_counter() - t0) * 1e3)
    res['stream_batched_two_timestamps_ms'] = round(stream_ms[-1], 1)
    res['stream_batched_rollover_ms'] = round(acc.get('_roll_over', 0.0) * 1e3, 1)
    res['stream_batched_triples'] = int(len(two))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
