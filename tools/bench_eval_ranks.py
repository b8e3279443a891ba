"""Sharded test-time evaluation: RENet.evaluate_stream_batched(process_group=...) at W = 1, 2, 4, 8 ranks (as many as the
machine has GPUs), one process per GPU over NCCL, on the ICEWS18- and GDELT-shaped streams of tools/bench_eval.py.  Prints
one JSON line.

    python tools/bench_eval_ranks.py [--datasets icews18,gdelt] [--num-k 1000] [--test-timestamps 3] [--reps 3]

One set of processes is spawned for the whole run; the world size alternates inside every repeat (W = 1, 2, 4, 8, then
again), ranks 0..W-1 evaluating over a group of their own while the others wait, every run from a fresh copy of the state
with the same seed.  Per test timestamp: the roll-over (_roll_over, per roll-over) and the scoring of the timestamp's triples
(_score_run: encode, rank call and host glue), each timed on the host clock between a device synchronise and a barrier of
the group at both ends, the max over ranks; ranges over the repeats.  Every W must give the W = 1 ranks and loss exactly,
or the script fails.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import socket
import sys
import time

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bench_eval                                   # noqa: E402


def _free_port():
    s = socket.socket(); s.bind(('127.0.0.1', 0)); p = s.getsockname()[1]; s.close()
    return p


def _timed(m, name, acc, group):
    """Wraps m.<name>: a device synchronise and a barrier of ``group`` at both ends of every call, host clock between."""
    fn = getattr(m, name)

    def wrapper(*a, **kw):
        torch.cuda.synchronize()
        if group is not None:
            dist.barrier(group=group)
        t0 = time.perf_counter()
        out = fn(*a, **kw)
        torch.cuda.synchronize()
        if group is not None:
            dist.barrier(group=group)
        acc.setdefault(name, []).append(time.perf_counter() - t0)
        return out
    setattr(m, name, wrapper)


def _worker(rank, world, port, args, out):
    os.environ['CUDA_VISIBLE_DEVICES'] = str(rank)          # rank r owns GPU r
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(0)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', 0))
    try:
        ws = [w for w in (1, 2, 4, 8) if w <= world]
        groups = {w: dist.new_group(list(range(w))) for w in ws}    # every rank creates every group, in the same order
        res = {}
        for ds in args.datasets.split(','):
            tkg, m, te, hist = bench_eval.setup(ds, args.num_k, args.test_timestamps)
            quads = tkg.quads
            gm = bench_eval.SeededGlobal(tkg.num_e)
            snap = bench_eval.snapshot(m)
            runs = {w: [] for w in ws}
            for rep in range(args.reps + 1):                      # the first round warms up
                for w in ws:
                    if rank < w:
                        bench_eval.restore(m, snap)
                        group = groups[w] if w > 1 else None
                        acc = {}
                        for name in ('_roll_over', '_score_run'):
                            _timed(m, name, acc, group)
                        torch.manual_seed(5)
                        r = m.evaluate_stream_batched(quads[te], hist[0], hist[1], gm, total_data=quads, process_group=group)
                        for name in ('_roll_over', '_score_run'):
                            delattr(m, name)
                        t = torch.tensor(acc['_roll_over'] + acc['_score_run'], dtype=torch.float64, device='cuda')
                        if group is not None:
                            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
                        n_roll = len(acc['_roll_over'])
                        if rep > 0:
                            runs[w].append(dict(rollover=t[:n_roll].tolist(), score=t[n_roll:].tolist(), ranks=r['ranks'],
                                                loss=r['loss']))
                    dist.barrier()
            if rank == 0:
                res[ds] = {'num_e': tkg.num_e, 'num_r': tkg.num_r, 'test_triples_per_timestamp':
                           [int((quads[te, 3] == t).sum()) for t in np.unique(quads[te, 3])], 'runs': runs}
        if rank == 0:
            out['res'] = res
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--datasets', default='icews18,gdelt')
    ap.add_argument('--num-k', type=int, default=1000)
    ap.add_argument('--test-timestamps', type=int, default=3)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_eval_ranks.py measures on GPUs; none is visible')
    world = min(torch.cuda.device_count(), 8)
    name, power = bench_eval.gpu_info()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), a, out), nprocs=world, join=True)
    raw = dict(out)['res']
    mgr.shutdown()
    res = {'device': name, 'power_limit_w': power, 'gpus': world, 'h': bench_eval.H, 'num_k': a.num_k, 'reps': a.reps}
    mismatch = []
    for ds, d in raw.items():
        ref = d['runs'][1][0]
        per_w = {}
        for w, runs in d['runs'].items():
            for r in runs:
                if not (np.array_equal(r['ranks'], ref['ranks']) and r['loss'] == ref['loss']):
                    mismatch.append((ds, w))
            rng = lambda xs: [round(min(xs) * 1e3, 1), round(max(xs) * 1e3, 1)]       # noqa: E731
            per_w[w] = {'rollover_ms_per_rollover': rng([float(np.mean(r['rollover'])) for r in runs]),
                        'scoring_ms_per_timestamp': rng([float(np.mean(r['score'])) for r in runs]),
                        'rollover_ms_each': [[round(x * 1e3, 1) for x in r['rollover']] for r in runs],
                        'scoring_ms_each': [[round(x * 1e3, 1) for x in r['score']] for r in runs]}
        res[ds] = {k: v for k, v in d.items() if k != 'runs'}
        res[ds]['per_world_size'] = per_w
    res['ranks_equal_to_w1'] = not mismatch
    print(json.dumps(res))
    if mismatch:
        raise SystemExit('ranks or loss differ from W = 1 at %s' % mismatch)


if __name__ == '__main__':
    main()
