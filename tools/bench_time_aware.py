"""Cost of the time-aware filter (evaluate_stream(time_aware=True)) on one GPU.  Prints one JSON line.

    python tools/bench_time_aware.py [--datasets icews18,gdelt] [--rounds 7] [--calls 20] [--stream-reps 3]
                                     [--compare-tree DIR --ab-rounds 3]

Per dataset shape (synthetic streams, h = 200; one test timestamp's rows, 2 per triple, against a FilterIndex /
TimeFilterIndex of the whole stream):
  (a) the rank kernel with one list (renet_decoder_rank, the static filter) against renet_decoder_rank_multi with two
      lists (static + time-aware), alternated --rounds times; each round times --calls back-to-back calls with CUDA events;
  (b) evaluate_stream_batched over the last 3 timestamps with time_aware off and on, alternated --stream-reps times, each
      from a fresh copy of the state: ms per timestamp without the roll-over (host clock after a device synchronise);
  (c) building the TimeFilterIndex (and, for scale, the FilterIndex) from an ICEWS18-sized stream of about 470 k
      quadruples, host clock.
--compare-tree DIR: the static call of (a) alone, in alternating processes importing renet_b200 from this tree and from DIR
(another checkout with its library built), --ab-rounds times each.  --static-only: one such process (used by the above)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = 'cuda:0'
H = 200


def _args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--datasets', default='icews18,gdelt')
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--calls', type=int, default=20)
    ap.add_argument('--stream-reps', type=int, default=3)
    ap.add_argument('--num-k', type=int, default=1000)
    ap.add_argument('--compare-tree', default=None)
    ap.add_argument('--ab-rounds', type=int, default=3)
    ap.add_argument('--static-only', action='store_true')
    ap.add_argument('--tree', default=ROOT)
    return ap.parse_args()


A = _args()
sys.path.insert(0, os.path.abspath(A.tree))

import numpy as np      # noqa: E402
import torch            # noqa: E402

from renet_b200 import synthetic                          # noqa: E402
from renet_b200.decoder import decoder_rank_counts        # noqa: E402
from renet_b200.inference import FilterIndex              # noqa: E402


def _dev(*arrays):
    return tuple(torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(DEV) for a in arrays)


def kernel_inputs(ds):
    """One test timestamp's rows of the synthetic stream (subject rows then object rows), their labels and exclusion
    lists: the static one and, where the tree has it, the time-aware one."""
    quads, num_e, _ = synthetic.make_quads(ds, seed=11)
    t = np.unique(quads[:, 3])[-3]
    q = quads[quads[:, 3] == t]
    n = len(q)
    gen = torch.Generator().manual_seed(7)
    x = (torch.randn(2 * n, 3 * H, generator=gen) * 0.2).to(DEV)
    w = (torch.randn(num_e, 3 * H, generator=gen) * 0.05).to(DEV)
    b = (torch.randn(num_e, generator=gen) * 0.1).to(DEV)
    lab = torch.from_numpy(np.concatenate((q[:, 0], q[:, 2]))).to(DEV)
    fix, rr = np.concatenate((q[:, 2], q[:, 0])), np.concatenate((q[:, 1], q[:, 1]))
    direction = np.concatenate((np.ones(n, bool), np.zeros(n, bool)))           # subject rows first
    lists = [(FilterIndex(quads), (fix, rr))]
    try:
        from renet_b200.inference import TimeFilterIndex
        lists.append((TimeFilterIndex(quads), (fix, rr, np.full(2 * n, t))))
    except ImportError:
        pass
    ex = []
    for idx, key in lists:
        b_ob, e_ob = idx.ranges('objects', *key)
        b_sb, e_sb = idx.ranges('subjects', *key)
        off = len(idx.col('objects'))
        col = np.concatenate((idx.col('objects'), idx.col('subjects')))
        ex.append(_dev(col, np.where(direction, b_sb + off, b_ob), np.where(direction, e_sb + off, e_ob)))
    return dict(x=x, w=w, b=b, lab=lab, ex=ex, rows=2 * n, num_e=num_e)


def time_calls(fn, calls):
    """ms per call over `calls` back-to-back calls, CUDA events."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / calls


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                           capture_output=True, text=True, timeout=60)
        power = float(q.stdout.strip().split('\n')[0])
    except (OSError, ValueError, subprocess.SubprocessError):
        power = None
    return name, power


def static_only(datasets, rounds, calls):
    out = {}
    with torch.no_grad():
        for ds in datasets:
            k = kernel_inputs(ds)
            fn = lambda: decoder_rank_counts(k['x'], k['w'], k['b'], k['lab'], k['ex'][0])   # noqa: E731
            for _ in range(3):
                fn()
            out[ds] = [round(time_calls(fn, calls), 4) for _ in range(rounds)]
    return out


def kernel_ab(ds, rounds, calls):
    from renet_b200.decoder import decoder_rank_counts_multi
    k = kernel_inputs(ds)
    one = lambda: decoder_rank_counts(k['x'], k['w'], k['b'], k['lab'], k['ex'][0])                # noqa: E731
    two = lambda: decoder_rank_counts_multi(k['x'], k['w'], k['b'], k['lab'], k['ex'])             # noqa: E731
    with torch.no_grad():
        l1, c1 = one()
        l2, c2 = two()
        assert torch.equal(l1, l2) and torch.equal(c1, c2[:, :4])
        res = {'one_list_ms': [], 'two_lists_ms': []}
        for _ in range(rounds):
            res['one_list_ms'].append(round(time_calls(one, calls), 4))
            res['two_lists_ms'].append(round(time_calls(two, calls), 4))
    lens = [(e[2] - e[1]).cpu().numpy() for e in k['ex']]
    res.update(rows=k['rows'], num_e=k['num_e'], mean_static_list=round(float(lens[0].mean()), 1),
               mean_time_list=round(float(lens[1].mean()), 1),
               rows_with_different_lists=int((lens[0] != lens[1]).sum()))
    return res


def stream_ab(ds, num_k, reps):
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    from bench_eval import SeededGlobal, restore, setup, snapshot, timed_method
    n_test = 3
    tkg, m, te, hist = setup(ds, num_k, n_test)
    quads = tkg.quads
    gm = SeededGlobal(tkg.num_e)
    snap = snapshot(m)

    def run(time_aware):
        restore(m, snap)
        acc = {}
        timed_method(m, '_roll_over', acc)
        torch.manual_seed(5)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = m.evaluate_stream_batched(quads[te], hist[0], hist[1], gm, total_data=quads, time_aware=time_aware)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        delattr(m, '_roll_over')
        return round((total - acc['_roll_over']) * 1e3 / n_test, 1), out

    _, base = run(False)
    _, ta = run(True)                                              # warm-up of both arms
    assert np.array_equal(base['ranks'], ta['ranks']) and base['loss'] == ta['loss']
    res = {'off_ms_per_timestamp': [], 'on_ms_per_timestamp': []}
    for _ in range(reps):
        res['off_ms_per_timestamp'].append(run(False)[0])
        res['on_ms_per_timestamp'].append(run(True)[0])
    res['mrr'] = {k: round(v['mrr'], 5) for k, v in ta['protocols'].items()}
    return res


def index_build(reps=3):
    from renet_b200.inference import TimeFilterIndex
    quads, _, _ = synthetic.make_quads('icews18', seed=11, num_timestamps=304)
    res = {'quads': int(len(quads)), 'time_filter_index_ms': [], 'filter_index_ms': []}
    for _ in range(reps):
        t0 = time.perf_counter()
        TimeFilterIndex(quads)
        res['time_filter_index_ms'].append(round((time.perf_counter() - t0) * 1e3, 1))
        t0 = time.perf_counter()
        FilterIndex(quads)
        res['filter_index_ms'].append(round((time.perf_counter() - t0) * 1e3, 1))
    return res


def main():
    if not torch.cuda.is_available():
        raise SystemExit('bench_time_aware.py measures on a GPU; none is visible')
    datasets = A.datasets.split(',')
    if A.static_only:
        print(json.dumps(static_only(datasets, A.rounds, A.calls)))
        return
    name, power = gpu_info()
    res = {'device': name, 'power_limit_w': power, 'h': H}
    for ds in datasets:
        res[ds] = {'kernel': kernel_ab(ds, A.rounds, A.calls), 'stream': stream_ab(ds, A.num_k, A.stream_reps)}
    res['index_build'] = index_build()
    if A.compare_tree:
        ab = {'this': {d: [] for d in datasets}, 'other': {d: [] for d in datasets}}
        for _ in range(A.ab_rounds):
            for arm, tree in (('this', A.tree), ('other', A.compare_tree)):
                cmd = [sys.executable, os.path.abspath(__file__), '--static-only', '--tree', tree, '--datasets', A.datasets,
                       '--rounds', str(A.rounds), '--calls', str(A.calls)]
                got = json.loads(subprocess.run(cmd, capture_output=True, text=True, check=True).stdout.strip().split('\n')[-1])
                for d in datasets:
                    ab[arm][d].extend(got[d])
        res['static_call_ms_this_vs_other_tree'] = ab
    print(json.dumps(res))


if __name__ == '__main__':
    main()
