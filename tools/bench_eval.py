"""Test-time scoring (reference model.py:365-419, test.py:98-150) on synthetic ICEWS18- and GDELT-shaped streams: the batched
path (RENet.evaluate_stream_batched) against the per-triple loop it replaces, on one GPU.  Prints one JSON line.

    python tools/bench_eval.py [--datasets icews18,gdelt] [--num-k 1000] [--old-triples 200] [--test-timestamps 3] [--reps 2]

The stream's last --test-timestamps timestamps are the test split; the per-entity histories start from everything before
them (init_history) and latest_time is the first test timestamp, as the test flow sets them up, so every later timestamp
rolls over once.
  (a) old: evaluate_filter (predict + the per-triple filter scan + two ranks) over the first --old-triples triples of the
      first test timestamp (no roll-over), in ms per triple;
  (b) new: evaluate_stream_batched over the whole test split, filtered: ms per timestamp in all, the roll-over per
      roll-over, and per timestamp the rest, batching + encode (_encode_queries, both directions) and the rank call
      (_rank_rows: renet_decoder_rank_multi with its inputs' uploads); each part ends in a device synchronise;
  (c) the rank kernel alone (renet_decoder_rank) on one timestamp's rows, timed with CUDA events: logical GEMM TFLOP/s of its
      two passes = 2 x 2 * rows * |E| * 3h over the call's time.
(a) and (b) alternate --reps times; every (b) starts from a fresh copy of the state.  The model has seeded parameters (h =
200); the global model is a seeded stand-in (the roll-over only needs its distributions); the streams are generated, so the
numbers describe the work's shape, not a dataset's accuracy."""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from renet_b200 import synthetic                  # noqa: E402
from renet_b200.decoder import decoder_rank        # noqa: E402
from renet_b200.inference import FilterIndex       # noqa: E402
from renet_b200.model import RENet                 # noqa: E402

DEV = 'cuda:0'
H = 200


class SeededGlobal:
    """Stand-in for the global model's predict(t, graph_dict, subject) -> (embedding [1,1,h], logits [1,1,|E|], prob)."""

    def __init__(self, num_e, seed=3):
        self.num_e, self.seed = num_e, seed

    def predict(self, t, graph_dict, subject=True):
        g = torch.Generator().manual_seed(self.seed + 7 * int(t) + (0 if subject else 100003))
        emb = 0.1 * torch.randn(1, 1, H, generator=g)
        logits = 2.0 * torch.randn(1, 1, self.num_e, generator=g)
        return emb, logits, torch.softmax(logits.view(-1), dim=0)


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                           capture_output=True, text=True, timeout=60)
        power = float(q.stdout.strip().split('\n')[0])
    except (OSError, ValueError, subprocess.SubprocessError):
        power = None
    return name, power


def setup(ds, num_k, n_test):
    tkg = synthetic.SyntheticTKG(ds, seed=11, h_dim=H)
    quads = tkg.quads
    times = np.unique(quads[:, 3])
    tr, te = np.flatnonzero(quads[:, 3] < times[-n_test]), np.flatnonzero(quads[:, 3] >= times[-n_test])
    torch.manual_seed(0)
    m = RENet(tkg.num_e, H, tkg.num_r, dropout=0, model=0, seq_len=10, num_k=num_k).to(DEV).eval()
    pick = lambda L, idx: [L[i] for i in idx]                                           # noqa: E731
    m.global_emb = dict(tkg.global_emb)
    m.graph_dict = dict(tkg.graph_dict)
    hist_tr = ((pick(tkg.s_hist, tr), pick(tkg.s_hist_t, tr)), (pick(tkg.o_hist, tr), pick(tkg.o_hist_t, tr)))
    hist = ((pick(tkg.s_hist, te), pick(tkg.s_hist_t, te)), (pick(tkg.o_hist, te), pick(tkg.o_hist_t, te)))
    m.init_history(quads[tr], hist_tr[0], hist_tr[1], [], ([], []), ([], []), quads[te], hist[0], hist[1])
    m.latest_time = torch.tensor(int(times[-n_test]))          # as test.py starts: the first test timestamp rolls nothing
    return tkg, m, te, hist


STATE = ('s_hist_test', 's_hist_test_t', 'o_hist_test', 'o_hist_test_t', 's_his_cache', 'o_his_cache', 's_his_cache_t',
         'o_his_cache_t', 'graph_dict', 'global_emb', 'latest_time')


def snapshot(m):
    return {k: copy.deepcopy(getattr(m, k)) for k in STATE}


def restore(m, snap):
    for k in STATE:
        setattr(m, k, copy.deepcopy(snap[k]))


def timed_method(m, name, acc):
    fn = getattr(m, name)

    def wrapper(*a, **kw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn(*a, **kw)
        torch.cuda.synchronize()
        acc[name] = acc.get(name, 0.0) + time.perf_counter() - t0
        return out
    setattr(m, name, wrapper)


def bench_dataset(ds, num_k, old_triples, n_test, reps):
    tkg, m, te, hist = setup(ds, num_k, n_test)
    quads = tkg.quads
    gm = SeededGlobal(tkg.num_e)
    snap = snapshot(m)
    t_first = quads[te[0], 3]
    first = te[quads[te, 3] == t_first]
    allt = torch.from_numpy(quads).to(DEV)
    out = {'num_e': tkg.num_e, 'num_r': tkg.num_r, 'num_k': num_k, 'test_timestamps': n_test,
           'test_triples_per_timestamp': [int((quads[te, 3] == t).sum()) for t in np.unique(quads[te, 3])]}

    def old():
        restore(m, snap)
        n = min(old_triples, len(first))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad():
            for i in first[:n]:
                k = int(np.flatnonzero(te == i)[0])
                m.evaluate_filter(torch.from_numpy(quads[i]).to(DEV), (hist[0][0][k], hist[0][1][k]), (hist[1][0][k], hist[1][1][k]),
                                  gm, allt)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / n

    def new():
        restore(m, snap)
        acc = {}
        for name in ('_roll_over', '_encode_queries', '_rank_rows'):
            timed_method(m, name, acc)
        torch.manual_seed(5)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.evaluate_stream_batched(quads[te], hist[0], hist[1], gm, total_data=quads)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        for name in ('_roll_over', '_encode_queries', '_rank_rows'):
            delattr(m, name)
        per = lambda s: round(s * 1e3 / n_test, 1)                                       # noqa: E731
        return dict(total=per(total), rollover_per_rollover=round(acc['_roll_over'] * 1e3 / (n_test - 1), 1),
                    total_without_rollover=per(total - acc['_roll_over']), encode=per(acc['_encode_queries']),
                    rank=per(acc['_rank_rows']),
                    other=per(total - acc['_roll_over'] - acc['_encode_queries'] - acc['_rank_rows']))

    old(), new()                                                 # warm up both paths
    olds, news = [], []
    for _ in range(reps):
        olds.append(round(old(), 2))
        news.append(new())
    out['old_ms_per_triple'] = olds
    out['old_triples_timed'] = min(old_triples, len(first))
    out['new_ms_per_timestamp'] = {k: [r[k] for r in news] for k in news[0]}
    n_first = len(first)
    out['old_ms_per_timestamp_extrapolated'] = [round(o * n_first, 0) for o in olds]

    # (c) the rank kernel alone on one timestamp's rows (subject and object rows: 2 per triple)
    rows = 2 * n_first
    gen = torch.Generator().manual_seed(7)
    x = (torch.randn(rows, 3 * H, generator=gen) * 0.2).to(DEV)
    lab = torch.randint(0, tkg.num_e, (rows,), generator=gen).to(DEV)
    fi = FilterIndex(quads)
    q = quads[first]
    b_o, e_o = fi.ranges('objects', q[:, 0], q[:, 1])
    b_s, e_s = fi.ranges('subjects', q[:, 2], q[:, 1])
    off = len(fi.col('objects'))
    col = np.concatenate((fi.col('objects'), fi.col('subjects')))
    ex = tuple(torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(DEV)
               for a in (col, np.concatenate((b_o, b_s + off)), np.concatenate((e_o, e_s + off))))
    w, b = m.linear.weight.detach(), m.linear.bias.detach()
    with torch.no_grad():
        decoder_rank(x, w, b, lab, ex)
        times = []
        for _ in range(max(reps, 5)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            decoder_rank(x, w, b, lab, ex)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
    flop = 2 * 2.0 * rows * tkg.num_e * 3 * H
    out['kernel_rows'] = rows
    out['kernel_ms'] = [round(t, 3) for t in times]
    out['kernel_gemm_tflops'] = [round(flop / (t * 1e-3) / 1e12, 1) for t in times]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--datasets', default='icews18,gdelt')
    ap.add_argument('--num-k', type=int, default=1000)
    ap.add_argument('--old-triples', type=int, default=200)
    ap.add_argument('--test-timestamps', type=int, default=3)
    ap.add_argument('--reps', type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_eval.py measures on a GPU; none is visible')
    name, power = gpu_info()
    res = {'device': name, 'power_limit_w': power, 'h': H}
    for ds in a.datasets.split(','):
        res[ds] = bench_dataset(ds, a.num_k, a.old_triples, a.test_timestamps, a.reps)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
