"""One pre-training epoch of the global model (reference pretrain.py:70-92) on synthetic ICEWS18- and GDELT-shaped streams,
the new path against the old one, on one GPU.  Prints one JSON line.

    python tools/bench_pretrain.py [--datasets icews18,gdelt] [--reps 3]

  (a) loss head, forward + backward: decoder_soft_cross_entropy against nn.Linear + the fp64 soft cross-entropy
      (utils.py:287-290), [1024,200] x [200,|E|] with true distributions as targets;
  (b) RENet_global.get_global_emb: the batched pass against a loop of predict calls (the per-timestamp definition of
      global_model.py:57-73), in eval mode and in train mode with dropout 0.5;
  (c) one epoch: the optimiser steps over batches of 1024 timestamps (DataParallelTrainer.step) plus the table.
Every arm is warmed up first; the arms alternate and each is timed 3 times (host clock after a device synchronise).
The stream lengths are the datasets' training timestamps (ICEWS18: 240, GDELT: 2,138); the streams are generated, so the
numbers say nothing about the datasets' accuracy, only about the work's shape."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from renet_b200 import synthetic                                  # noqa: E402
from renet_b200.decoder import decoder_soft_cross_entropy         # noqa: E402
from renet_b200.global_model import RENet_global, gru_final_hidden  # noqa: E402
from renet_b200.parallel import DataParallelTrainer              # noqa: E402

DEV = 'cuda:0'
H = 200
BATCH = 1024
TIMESTAMPS = {'icews18': 240, 'gdelt': 2138}


def true_distribution(quads, num_e):
    """Restatement of the reference's get_true_distribution (utils.py:292-324): a triple is counted before the timestamp
    change is seen, so each timestamp's first triple lands in the previous row; every row but the last is normalised."""
    t = quads[:, 3]
    prev = np.concatenate(([0], t[:-1]))
    change = (t != prev).astype(np.int64)
    row = np.cumsum(change) - change
    n_rows = int(change.sum()) + 1
    out = []
    for col in (0, 2):
        m = np.zeros((n_rows, num_e))
        np.add.at(m, (row, quads[:, col]), 1.0)
        m[:-1] /= m[:-1].sum(axis=1, keepdims=True)
        out.append(m)
    return out


def old_soft_cross_entropy(pred, soft_targets):
    logp = F.log_softmax(pred.double(), dim=1)
    return torch.mean(torch.sum(-soft_targets.double() * logp, 1))


def old_forward(m, t_list, true_prob_s, true_prob_o, graph_dict):
    """RENet_global.forward of the parent revision (subject direction): nn.Linear + the fp64 soft cross-entropy."""
    t_host = np.asarray(t_list.tolist(), dtype=np.int64)
    idx = np.argsort(-t_host, kind='stable')
    X, lens = m.aggregator.rows(t_host[idx], m.ent_embeds, graph_dict, False)
    s_q = gru_final_hidden(m.encoder_global, X, lens)
    s_q = torch.cat((s_q, torch.zeros(len(t_host) - s_q.shape[0], m.h_dim, device=s_q.device)), dim=0)
    return old_soft_cross_entropy(m.linear_s(s_q), true_prob_o[torch.from_numpy(idx).to(true_prob_o.device)])


def old_global_emb(m, t_list, graph_dict):
    """get_global_emb of the parent revision: one predict call per timestamp."""
    times = list(graph_dict.keys())
    unit = times[1] - times[0]
    out, prev = {}, 0
    for t in t_list:
        if t == 0:
            continue
        out[prev] = m.predict(t, graph_dict)[0].detach()
        prev = t
    out[t_list[-1]] = m.predict(t_list[-1] + unit, graph_dict)[0].detach()
    return out


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def ab(arms, reps):
    """{name: [seconds] * reps}: one warm-up call per arm, then the arms alternate."""
    for fn in arms.values():
        timed(fn)
    res = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            res[k].append(round(timed(fn) * 1e3, 3))
    return res


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                           capture_output=True, text=True, timeout=60)
        power = float(q.stdout.strip().split('\n')[0])
    except (OSError, ValueError, subprocess.SubprocessError):
        power = None
    return name, power


def bench_dataset(ds, reps):
    T = TIMESTAMPS[ds]
    quads, num_e, num_r = synthetic.make_quads(ds, seed=11, num_timestamps=T)
    gd = synthetic.build_graph_dict(quads, num_r)
    train_times = sorted(gd)
    ps, po = (torch.from_numpy(a).to(DEV) for a in true_distribution(quads, num_e))
    out = {'num_e': num_e, 'timestamps': T, 'instance_nodes': None}

    # (a) loss head
    gen = torch.Generator().manual_seed(0)
    rows = torch.randint(0, T, (BATCH,), generator=gen)
    x = (torch.randn(BATCH, H, generator=gen) * 0.5).to(DEV).requires_grad_(True)
    lin = torch.nn.Linear(H, num_e).to(DEV)
    P = po[rows.to(DEV)]

    def fused():
        decoder_soft_cross_entropy(x, lin.weight, lin.bias, P).backward()

    def torch_head():
        old_soft_cross_entropy(lin(x), P).backward()
    out['loss_head_ms'] = ab({'fused': fused, 'linear_fp64': torch_head}, reps)

    # (b) the table
    torch.manual_seed(0)
    m = RENet_global(num_e, H, num_r, dropout=0.5, model=3, seq_len=10, num_k=10, maxpool=1).to(DEV)
    sizes = {t: g.number_of_nodes() for t, g in gd.items()}
    times = list(gd)
    out['instance_nodes'] = int(sum(sum(sizes[u] for u in times[max(0, i - 10):i]) for i in range(1, len(times))))
    tab = {}
    for mode in ('eval', 'train'):
        m.train(mode == 'train')
        with torch.no_grad():
            tab[mode] = ab({'batched': lambda: m.get_global_emb(train_times, gd),
                            'predict_loop': lambda: old_global_emb(m, train_times, gd)}, reps)
    out['global_emb_ms'] = tab
    m.eval()
    with torch.no_grad():
        a, b = m.get_global_emb(train_times, gd), old_global_emb(m, train_times, gd)
    out['global_emb_max_abs_diff_eval'] = float(max((a[k] - b[k]).abs().max() for k in b))

    # (c) one epoch: optimiser steps over shuffled batches of timestamps, then the table (pretrain.py:70-92)
    m.train()
    tr = DataParallelTrainer(m, lr=1e-3, weight_decay=0.0, grad_norm=1.0)
    perm = np.random.RandomState(0).permutation(T)
    batches = [perm[i:i + BATCH] for i in range(0, T, BATCH)]

    def epoch(new):
        for sel in batches:
            tb = torch.from_numpy(np.asarray(train_times)[sel]).to(DEV)
            s, o = ps[torch.from_numpy(sel).to(DEV)], po[torch.from_numpy(sel).to(DEV)]
            if new:
                tr.step(lambda: m(tb, s, o, gd), local_weight=len(sel))
            else:
                tr.step(lambda: old_forward(m, tb, s, o, gd), local_weight=len(sel))
            tr.zero_grad()
        with torch.no_grad():
            (m.get_global_emb if new else lambda tl, g: old_global_emb(m, tl, g))(train_times, gd)
    out['epoch_ms'] = ab({'new': lambda: epoch(True), 'old': lambda: epoch(False)}, reps)
    out['steps_per_epoch'] = len(batches)
    tr.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--datasets', default='icews18,gdelt')
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_pretrain: needs a CUDA device')
    name, power = gpu_info()
    res = {'device': name, 'power_limit_w': power, 'batch': BATCH, 'h': H}
    for ds in args.datasets.split(','):
        res[ds] = bench_dataset(ds, args.reps)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
