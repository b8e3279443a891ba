"""One test-time roll-over's candidate scoring (reference model.py:222-279) on synthetic ICEWS18- and GDELT-shaped streams,
the batched path against the per-entity loop it replaces, on one GPU.  Prints one JSON line.

    python tools/bench_rollover.py [--datasets icews18,gdelt] [--num-k 1000] [--old-picks 16] [--reps 3]

  (a) new: RENet.pred_r_topk for the distinct picks of num_k samples, subject and object direction together (what
      _roll_over runs before its host steps), including the history batching and the device-to-host copy of the lists;
  (b) old: pred_r_rank2 + torch.topk + the copy to the host for the first --old-picks picks of each direction, reported
      as ms per pick on that subset (not extrapolated to num_k);
  (c) the fused top-k alone (renet_decoder_group_topk) on one chunk of ROLLOVER_SEQ_BUDGET rows, timed with CUDA events:
      GEMM TFLOP/s of its two passes = 2 x 2 * rows * |E| * 3h over the call's time.
The model has seeded parameters (h = 200) and the sampling distribution is a seeded softmax over the entities; the
streams are generated, so the numbers describe the work's shape, not a dataset's accuracy."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from renet_b200 import synthetic                                  # noqa: E402
from renet_b200.decoder import decoder_group_topk                # noqa: E402
from renet_b200.inference import ROLLOVER_SEQ_BUDGET  # noqa: E402
from renet_b200.model import RENet                                # noqa: E402

DEV = 'cuda:0'
H = 200


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                           capture_output=True, text=True, timeout=60)
        power = float(q.stdout.strip().split('\n')[0])
    except (OSError, ValueError, subprocess.SubprocessError):
        power = None
    return name, power


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def setup(ds, num_k):
    tkg = synthetic.SyntheticTKG(ds, seed=11, h_dim=H)
    torch.manual_seed(0)
    m = RENet(tkg.num_e, H, tkg.num_r, dropout=0, model=0, seq_len=10, num_k=num_k).to(DEV).eval()
    m.global_emb = tkg.global_emb
    m.graph_dict = dict(tkg.graph_dict)
    m.init_history(tkg.quads, (tkg.s_hist, tkg.s_hist_t), (tkg.o_hist, tkg.o_hist_t), [], ([], []), ([], []))
    gen = torch.Generator().manual_seed(5)
    prob = torch.softmax(2.0 * torch.randn(tkg.num_e, generator=gen), dim=0)
    torch.manual_seed(6)
    picks = {s: torch.distributions.categorical.Categorical(prob).sample(torch.Size([num_k])) for s in (True, False)}
    return tkg, m, prob, picks


def bench_dataset(ds, num_k, old_picks, reps):
    tkg, m, prob, picks = setup(ds, num_k)
    R, N = tkg.num_r, tkg.num_e
    out = {'num_e': N, 'num_r': R, 'num_k': num_k}

    def new():
        for subject in (True, False):
            uniq, inverse = torch.unique(picks[subject], return_inverse=True)
            v, c = m.pred_r_topk(uniq, prob[uniq], num_k, subject=subject)
            v.cpu()[inverse.cpu()], c.cpu()[inverse.cpu()]

    def old():
        for subject in (True, False):
            for e in picks[subject][:old_picks].tolist():
                joint = float(prob[e]) * m.pred_r_rank2(torch.full((R,), e, dtype=torch.long), torch.arange(R), subject=subject)
                tp, ti = torch.topk(joint.view(-1), num_k, sorted=False)
                tp.cpu(), ti.cpu()

    out['distinct_picks'] = [int(torch.unique(picks[s]).numel()) for s in (True, False)]
    with torch.no_grad():
        timed(new)
        timed(old)
        new_ms, old_ms = [], []
        for _ in range(reps):
            new_ms.append(round(timed(new) * 1e3, 1))
            old_ms.append(round(timed(old) * 1e3 / (2 * old_picks), 2))
    out['new_ms_both_directions'] = new_ms
    out['old_ms_per_pick_on_subset'] = old_ms
    out['old_subset_picks_per_direction'] = old_picks

    # (c) the fused kernel on one chunk
    per = max(1, ROLLOVER_SEQ_BUDGET // R)
    rows = per * R
    gen = torch.Generator().manual_seed(7)
    x = (torch.randn(rows, 3 * H, generator=gen) * 0.2).to(DEV)
    rw = (torch.rand(rows, generator=gen) * 1e-3).to(DEV)
    order = 0
    w, b = m.linear.weight.detach(), m.linear.bias.detach()
    with torch.no_grad():
        decoder_group_topk(x, w, b, rw, R, num_k, order)
        times = []
        for _ in range(max(reps, 3)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            decoder_group_topk(x, w, b, rw, R, num_k, order)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
    flop = 2 * 2.0 * rows * N * 3 * H
    out['kernel_chunk_rows'] = rows
    out['kernel_ms'] = [round(t, 3) for t in times]
    out['kernel_gemm_tflops'] = [round(flop / (t * 1e-3) / 1e12, 1) for t in times]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--datasets', default='icews18,gdelt')
    ap.add_argument('--num-k', type=int, default=1000)
    ap.add_argument('--old-picks', type=int, default=16)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_rollover.py measures on a GPU; none is visible')
    name, power = gpu_info()
    res = {'device': name, 'power_limit_w': power, 'h': H}
    for ds in a.datasets.split(','):
        res[ds] = bench_dataset(ds, a.num_k, a.old_picks, a.reps)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
