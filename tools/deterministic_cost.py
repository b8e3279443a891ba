#!/usr/bin/env python
"""Cost of the deterministic mode on the training step: bench.py's training region with and without
torch.use_deterministic_algorithms(True), alternated in fresh processes.

    python tools/deterministic_cost.py [--repeats 3] [--steps 40] [--warmup 5] [--dropout 0.0]

bench.py itself is run unchanged.  For the deterministic arm the flag is set in the process before bench.py starts, so
renet_b200._lib passes it on to the library at the first kernel call; CUBLAS_WORKSPACE_CONFIG is set for that process
as torch requires under the flag.  Prints one JSON line: the card's name and power limit (read in the same run) and,
per arm, the ms per step and the forward / backward phase times of every repeat.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BENCH = os.path.join(ROOT, 'bench.py')
LAUNCH = ('import runpy, sys, torch\n'
          'torch.use_deterministic_algorithms(%s)\n'
          'sys.argv = [%r] + sys.argv[1:]\n'
          'runpy.run_path(%r, run_name="__main__")\n')


def run_arm(deterministic, args):
    code = LAUNCH % (deterministic, BENCH, BENCH)
    env = dict(os.environ)
    if deterministic:
        env['CUBLAS_WORKSPACE_CONFIG'] = ':4096:8'
    cmd = [sys.executable, '-c', code, '--gpus', '1', '--mode', 'train', '--steps', str(args.steps), '--warmup',
           str(args.warmup), '--dropout', str(args.dropout)]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith('{')]
    if r.returncode != 0 or not lines:
        raise SystemExit('bench.py failed (deterministic=%s):\n%s' % (deterministic, r.stderr[-3000:]))
    line = json.loads(lines[-1])
    return {'ms_per_step': line['ms_per_step'], 'forward_ms': line['train']['forward_ms'],
            'backward_ms': line['train']['backward_ms']}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--dropout', type=float, default=0.0)
    args = ap.parse_args()
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True).stdout.strip()
    arms = {'default': [], 'deterministic': []}
    for _ in range(args.repeats):
        arms['default'].append(run_arm(False, args))
        arms['deterministic'].append(run_arm(True, args))
    print(json.dumps({'gpu': card, 'steps': args.steps, 'warmup': args.warmup, 'dropout': args.dropout, **arms}))


if __name__ == '__main__':
    main()
