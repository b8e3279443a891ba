"""Cost of history length on one GPU: the training step, the encode of evaluate_observed and renet_gru_fwd / _bwd alone at
seq_len 10, 20, 32 and 64, on a synthetic ICEWS18-shaped stream.  Prints one JSON line.

    python tools/bench_seq_len.py [--lengths 10,20,32,64] [--reps 5] [--steps 5]

The stream has 2 x 64 + 10 timestamps, so the samples of the last third (where the batches come from) have full histories
at every length.  Per length: RENet(h = 200, dropout 0.5, seq_len = L) with histories from build_history(history_len=L).
  * train: one step = both directions' forward and backward plus torch's Adam, batch 1024 (HistoryViews through the
    device batcher, as bench.py's training region), host clock around --steps steps ending in a device synchronise;
  * encode: RENet._encode_queries of evaluate_observed for every subject-side query of the last timestamp, over
    observed_history(history_len=L) windows (eval mode, no autograd);
  * gru_fwd / gru_bwd: renet_gru_fwd_dropout / renet_gru_bwd_dropout alone on the subject side of one training batch,
    CUDA events over 20 launches each.
The lengths alternate inside each of --reps rounds; reported are the median and the range over the rounds.  Also
reported: the batch's read-out rows S and sequences Q, the GRU's forward and backward workspace bytes for that batch,
and the peak memory torch allocated over a training step.  The card's name and power limit are read in the same run."""
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
from renet_b200 import _lib, synthetic               # noqa: E402
from renet_b200.hoststore import GraphStore, HistoryStore  # noqa: E402
from renet_b200.model import RENet                   # noqa: E402


class Arm:
    """Everything one history length needs, built once."""

    def __init__(self, tkg, gs, L, dev):
        self.L = L
        q = tkg.quads
        sh, sht, oh, oht = synthetic.build_history(q, history_len=L)
        self.stores = (HistoryStore(sh, sht, q[:, 0], gs, reverse=False), HistoryStore(oh, oht, q[:, 2], gs, reverse=True))
        self.sel = [tkg.batch_indices(i, 1024) for i in range(4)]
        torch.manual_seed(0)
        self.m = RENet(tkg.num_e, 200, tkg.num_r, dropout=0.5, seq_len=L).to(dev).train()
        self.m.global_emb = tkg.global_emb
        self.opt = torch.optim.Adam(self.m.parameters(), lr=1e-3)
        self.batches = [torch.from_numpy(q[s]).long().to(dev) for s in self.sel]
        self.gs, self.i = gs, 0
        times = np.unique(q[:, 3])
        test = q[q[:, 3] == times[-1]]
        self.obs = synthetic.observed_history(q, test[:, 0], test[:, 3], True, history_len=L)
        self.test = test

    def step(self):
        k = self.i % len(self.sel)
        self.i += 1
        vs, vo = (st.select(self.sel[k]) for st in self.stores)
        self.opt.zero_grad()
        loss = self.m(self.batches[k], vs, vo, self.gs, subject=True) + self.m(self.batches[k], vs, vo, self.gs, subject=False)
        loss.backward()
        self.opt.step()

    def encode(self):
        m = self.m
        m.eval()
        with torch.no_grad():
            (hist, has) = m._observed_histories(self.test[:, 0], self.obs, 's_history', self.gs.graph_dict, m.global_emb)
            m._encode_queries(self.test[:, 0], self.test[:, 1], has, True, history=hist,
                              graphs=(self.gs.graph_dict, m.global_emb))
        m.train()


def gru_alone(arm, dev, reps=20):
    """renet_gru_fwd_dropout / renet_gru_bwd_dropout on the subject side of the arm's first batch: (fwd ms, bwd ms, S, Q,
    forward workspace bytes, backward workspace bytes)."""
    from renet_b200.hoststore import assemble_view
    L, P = _lib.lib(), _lib.ptr
    m, h = arm.m, 200
    hb = assemble_view(arm.stores[0].select(arm.sel[0]), dev)
    S, Q, T = hb.S, hb.num_seq, 256
    bs = hb.batch_sizes
    hbs, ml = bs.ctypes.data_as(_lib.ctypes.c_void_p), len(bs)
    g = torch.Generator(device=dev).manual_seed(1)
    H2 = torch.randn(S, h, device=dev, generator=g)
    readout = torch.arange(S, dtype=torch.int32, device=dev)
    row_glob = torch.randint(0, T, (S,), device=dev, dtype=torch.int32, generator=g)
    glob = torch.randn(T, h, device=dev, generator=g)
    seq_s = torch.randint(0, m.in_dim, (Q,), device=dev, dtype=torch.int32, generator=g)
    seq_r = torch.randint(0, m.num_rels, (Q,), device=dev, dtype=torch.int32, generator=g)
    e4, e3 = m.encoder, m.encoder_r
    W = [P(t) for t in (e4.weight_ih_l0, e4.weight_hh_l0, e4.bias_ih_l0, e4.bias_hh_l0, e3.weight_ih_l0, e3.weight_hh_l0,
                        e3.bias_ih_l0, e3.bias_hh_l0)]
    WB = [W[0], W[1], W[4], W[5]]
    fb = int(L.renet_gru_dropout_workspace_bytes_len(S, Q, T, h, ml))
    bb = int(L.renet_gru_bwd_dropout_workspace_bytes_len(S, Q, T, h, ml))
    ws, bws = torch.empty(fb // 4 + 32, device=dev), torch.empty(bb // 4 + 32, device=dev)
    hn4, hn3 = torch.empty(Q, h, device=dev), torch.empty(Q, h, device=dev)
    dhn4, dhn3 = torch.randn(Q, h, device=dev, generator=g), torch.randn(Q, h, device=dev, generator=g)
    dH2 = torch.empty(S, h, device=dev)
    d_ent, d_rel, d_glob = (torch.zeros(n, h, device=dev) for n in (m.in_dim, m.num_rels, T))
    grads = [torch.zeros_like(p) for p in (e4.weight_ih_l0, e4.weight_hh_l0, e4.bias_ih_l0, e4.bias_hh_l0, e3.weight_ih_l0,
                                           e3.weight_hh_l0, e3.bias_ih_l0, e3.bias_hh_l0)]
    ent, rel, st = P(m.ent_embeds), P(m.rel_embeds), _lib.stream()

    def fwd():
        _lib.check(L.renet_gru_fwd_dropout(P(H2), P(readout), P(row_glob), P(glob), ent, rel, P(hb.row_seq), P(seq_s), P(seq_r),
                                           P(hb.graph.seq_len_dev), P(hb.seq_start), hbs, ml, *W, P(hn4), P(hn3), S, Q, T, h,
                                           0.5, 7, P(ws), fb, st), 'renet_gru_fwd_dropout')

    def bwd():
        _lib.check(L.renet_gru_bwd_dropout(P(H2), P(readout), P(row_glob), P(glob), ent, rel, P(hb.row_seq), P(seq_s),
                                           P(seq_r), P(hb.graph.seq_len_dev), P(hb.seq_start), hbs, ml, *WB, P(dhn4), P(dhn3),
                                           P(dH2), P(d_ent), P(d_rel), P(d_glob), *[P(x) for x in grads], S, S, Q, T, h, 0.5,
                                           7, P(ws), P(bws), bb, st), 'renet_gru_bwd_dropout')
    out = []
    for fn in (fwd, bwd):
        fn()
        torch.cuda.synchronize()
        b, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        b.record()
        for _ in range(reps):
            fn()
        e.record()
        torch.cuda.synchronize()
        out.append(b.elapsed_time(e) / reps)
    return out + [S, Q, fb, bb]


def timed(fn, n=1):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lengths', default='10,20,32,64')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--steps', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_seq_len needs a GPU'
    dev = torch.device('cuda:0')
    name, power = gpu_info()
    lengths = [int(x) for x in args.lengths.split(',')]
    tkg = synthetic.SyntheticTKG('icews18', seed=999, num_timestamps=2 * max(lengths) + 10)
    gs = GraphStore(tkg.graph_dict)
    arms = [Arm(tkg, gs, L, dev) for L in lengths]
    samples = {L: {'train_ms': [], 'encode_ms': [], 'gru_fwd_ms': [], 'gru_bwd_ms': []} for L in lengths}
    extra = {}
    for a in arms:                                            # warm-up, and the memory figures
        a.step()
        a.encode()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        a.step()
        torch.cuda.synchronize()
        extra[a.L] = {'train_peak_bytes': int(torch.cuda.max_memory_allocated(dev))}
    for _ in range(args.reps):
        for a in arms:
            s = samples[a.L]
            s['train_ms'].append(timed(a.step, args.steps))
            s['encode_ms'].append(timed(a.encode))
            f, b, S, Q, fb, bb = gru_alone(a, dev)
            s['gru_fwd_ms'].append(f)
            s['gru_bwd_ms'].append(b)
            extra[a.L].update(S=S, Q=Q, gru_fwd_ws_bytes=fb, gru_bwd_ws_bytes=bb, encode_queries=len(a.test))
    res = {'gpu': name, 'power_limit_w': power, 'reps': args.reps, 'steps': args.steps, 'lengths': {}}
    for L in lengths:
        r = dict(extra[L])
        for k, v in samples[L].items():
            r[k] = {'median': round(float(np.median(v)), 3), 'min': round(float(np.min(v)), 3), 'max': round(float(np.max(v)), 3)}
        res['lengths'][str(L)] = r
    print(json.dumps(res))


if __name__ == '__main__':
    main()
