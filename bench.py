#!/usr/bin/env python
"""bench.py -- edge-messages/s of the RGCN aggregate on ICEWS18-shaped history graphs (BASELINE.json).

    python bench.py --gpus N --steps K --warmup W            # our arm (CUDA kernels through the C-ABI)
    python bench.py --impl reference --gpus N --steps K ...  # the reference's CPU path (oracle port)
    python bench.py --steps K --dump-outputs DIR             # also write the last timed step's outputs as DIR/*.npy

A "step" is one training step's worth of the hot path over one batch of 1024 synthetic quadruples:
both directions (train.py:136-137) x both RGCN layers (Aggregator.py:136-137) over the batched history
graphs, i.e. 4 fused-layer passes = 2*(E_subj + E_obj) edge-messages (SURVEY.md section 8(d)).

  value       device-timed: graphs already resident in HBM, K steps between CUDA events, max over ranks
  e2e         the same work through the public API (RGCNAggregator / RENet.encode) from HOST inputs
              (history lists, graph_dict, triplets): host batching + pinned H2D + kernels + D2H of the
              GRU outputs, wall clock
  roofline    the fused gather kernel alone, CUDA events around every launch in a second timed region
  cpu_baseline  the reference's own op sequence (index_select -> bmm -> index_add, RGCN.py:79-94) on the
              host cores, bounded sample

L2 hygiene: the timed steps rotate over a pool of distinct pre-built batches whose combined footprint
(graph arrays + layer outputs) exceeds 2x the 50 MB L2 of an H100 ("l2": "rotating-pool" in config).
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

# torchrun exports OMP_NUM_THREADS=1 for every rank unless the application tunes it ("please further tune the variable
# for optimal performance in your application as needed").  Measured on a 2-GPU box: with 1 the end-to-end loop ran at
# 6.75 ms/step per rank, with 8 at 1.52 ms/step; the kernels' own numbers do not depend on it.  Must happen before numpy /
# torch load their OpenMP runtime.
def _rank_cpu_budget():
    """CPUs this rank may reasonably use: (cgroup quota or visible CPUs) / ranks on this host."""
    n = os.cpu_count() or 1
    try:
        _q, _per = open('/sys/fs/cgroup/cpu.max').read().split()
        if _q != 'max':
            n = min(n, max(1, int(float(_q) / float(_per))))
    except Exception:
        pass
    return max(1, n // max(1, int(os.environ.get('LOCAL_WORLD_SIZE', os.environ.get('WORLD_SIZE', '1')))))


if os.environ.get('OMP_NUM_THREADS') == '1' and 'LOCAL_RANK' in os.environ:
    os.environ['OMP_NUM_THREADS'] = str(max(1, min(8, _rank_cpu_budget() // 3)))

# Under a cgroup CPU quota far below the visible core count (16-24 CPUs of 128 on the GPU boxes) an OpenMP pool sized by
# the core count only burns the quota in spin-waits: size it by the quota.
if 'OMP_NUM_THREADS' not in os.environ:
    try:
        _q, _per = open('/sys/fs/cgroup/cpu.max').read().split()
        if _q != 'max':
            os.environ['OMP_NUM_THREADS'] = str(max(1, int(float(_q) / float(_per))))
    except Exception:
        pass

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

H_DIM, NUM_BASES, BATCH = 200, 100, 1024
METRIC = 'rgcn_aggregate_edge_messages_per_sec'
UNIT = 'edge-msg/s'
WORKLOADS = {
    # name: (synthetic preset, timestamps, description) -- BASELINE.json configs[1] / configs[2] / configs[4]
    'icews18': ('icews18', 240, 'ICEWS18-shaped synthetic TKG (23033 ent, 256 rel, 240 timestamps), n_hidden=200 num_bases=100 batch=1024'),
    'gdelt': ('gdelt', 2138, 'GDELT-shaped synthetic TKG (7691 ent, 240 rel, 2138 timestamps; ~2100 components per batch), n_hidden=200 '
                             'num_bases=100 seq-len=10 batch=1024'),
    'synth1m': (None, 250, 'synthetic TKG shard: 1M entities / 500 relations / 250 timesteps per GPU, avg in-degree 32 (N=1M nodes, '
                           'E=32M directed edges per GPU), n_hidden=200 num_bases=100; aggregate + GRU only'),
}
WORKLOAD = WORKLOADS['icews18'][2]


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--impl', default='ours', choices=['ours', 'reference'])
    ap.add_argument('--workload', default='icews18', choices=sorted(WORKLOADS))
    ap.add_argument('--timestamps', type=int, default=None)
    ap.add_argument('--synth-nodes', type=int, default=1_000_000, help='synth1m: nodes per GPU (edges = 32 x nodes)')
    ap.add_argument('--pool', type=int, default=8, help='distinct pre-built batches the timed steps rotate over')
    ap.add_argument('--no-cpu-baseline', action='store_true')
    ap.add_argument('--no-e2e', action='store_true')
    ap.add_argument('--host-batcher', action='store_true', help='e2e with the all-host C++ batcher instead of the device batcher')
    ap.add_argument('--mode', default='aggregate', choices=['aggregate', 'train'],
                    help="aggregate: the BASELINE metric line (it also carries a 'train' object); train: only the training-step region, "
                         "as the line's value")
    ap.add_argument('--no-train', action='store_true', help='skip the training-step region of the default line')
    ap.add_argument('--dropout', type=float, default=0.0, help='dropout of the training-step region (reference default 0.5)')
    ap.add_argument('--dump-outputs', metavar='DIR', default=None,
                    help='after the timed steps, write what the last timed step computed as DIR/<name>.npy (float32)')
    return ap.parse_args()


def algorithmic_bytes(N, E, R2):
    """SURVEY.md section 8(d), fp32 features, int32 indices, per fused-gather launch:
    E*(4h + 12) + N*(4h loop read + 4h write + 4 norm) + R2*(h*h/nb)*4."""
    return E * (4 * H_DIM + 12) + N * (8 * H_DIM + 4) + R2 * (H_DIM * H_DIM // NUM_BASES) * 4


def _cpu_quota():
    """CPUs the container may actually use (cgroup v2 cpu.max), or None: `cores` threads are started, the quota caps them."""
    try:
        q, per = open('/sys/fs/cgroup/cpu.max').read().split()
        return None if q == 'max' else round(float(q) / float(per), 2)
    except Exception:
        return None


class ClockSampler:
    """SM clock and throttle reasons sampled DURING the timed region.  NVML is
    polled in-process every few ms (a fresh `nvidia-smi -lms` takes longer to start than the timed region
    lasts); falls back to one nvidia-smi query if pynvml is unavailable."""

    def __init__(self, index):
        self.index, self.sm, self.reasons, self.max_mhz = index, [], set(), None
        self._stop = threading.Event()
        self.t = None

    def start(self):
        try:
            import pynvml
            pynvml.nvmlInit()
            vis = os.environ.get('CUDA_VISIBLE_DEVICES')
            idx = int(vis.split(',')[self.index]) if vis and vis.split(',')[self.index].isdigit() else self.index
            h = pynvml.nvmlDeviceGetHandleByIndex(idx)
            self.max_mhz = float(pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM))
            bits = {'hw_slowdown': getattr(pynvml, 'nvmlClocksEventReasonHwSlowdown', 0x8),
                    'hw_thermal_slowdown': getattr(pynvml, 'nvmlClocksEventReasonHwThermalSlowdown', 0x40),
                    'sw_thermal_slowdown': getattr(pynvml, 'nvmlClocksEventReasonSwThermalSlowdown', 0x20),
                    'sw_power_cap': getattr(pynvml, 'nvmlClocksEventReasonSwPowerCap', 0x4)}

            def poll():
                get_reasons = getattr(pynvml, 'nvmlDeviceGetCurrentClocksEventReasons',
                                      getattr(pynvml, 'nvmlDeviceGetCurrentClocksThrottleReasons', None))
                while not self._stop.is_set():
                    try:
                        self.sm.append(float(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)))
                        if get_reasons is not None:
                            r = int(get_reasons(h))
                            for n, b in bits.items():
                                if r & b:
                                    self.reasons.add(n)
                    except Exception:
                        pass
                    time.sleep(0.002)
            self.t = threading.Thread(target=poll, daemon=True)
            self.t.start()
        except Exception:
            self.t = None

    def stop(self):
        if self.t is not None:
            self._stop.set()
            self.t.join(timeout=5)
            if not self.t.is_alive():
                # leave nothing of NVML behind in this process: the end-to-end loop that follows is bound by CUDA API
                # calls on the host, and an initialised NVML client shares driver locks with them
                try:
                    import pynvml
                    pynvml.nvmlShutdown()
                except Exception:
                    pass
            return {'sm_mhz': float(np.median(self.sm)) if self.sm else None, 'sm_max_mhz': self.max_mhz,
                    'samples': len(self.sm), 'reasons': sorted(self.reasons), 'source': 'nvml, polled every 2 ms'}
        try:
            out = subprocess.run(['nvidia-smi', '-i', str(self.index), '--query-gpu=clocks.sm,clocks.max.sm',
                                  '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=10).stdout
            f = [float(x) for x in out.strip().split(',')]
            return {'sm_mhz': f[0], 'sm_max_mhz': f[1], 'samples': 1, 'reasons': [], 'source': 'nvidia-smi after the run'}
        except Exception:
            return {'sm_mhz': None, 'sm_max_mhz': None, 'samples': 0, 'reasons': ['clock query unavailable']}


def measured_peak_gbs():
    p = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(p):
        try:
            return float(json.load(open(p))['hbm_gbs']), 'measured (MEASURED_PEAKS.json hbm_gbs)'
        except Exception:
            pass
    return 3350.0, 'fallback (H100 SXM data sheet: 3.35 TB/s HBM3, not measured)'


def measured_peak_tf32():
    """Dense TF32 tensor peak = half the measured bf16 cuBLAS throughput (MEASURED_PEAKS.json), else the H100 SXM data sheet."""
    p = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(p):
        try:
            return float(json.load(open(p))['bf16_tflops']) / 2, 'measured (MEASURED_PEAKS.json bf16_tflops / 2: TF32 runs at half the bf16 rate)'
        except Exception:
            pass
    return 495.0, 'fallback (H100 SXM data sheet: 495 TFLOP/s dense TF32, not measured)'


def ncu_traffic():
    p = os.path.join(ROOT, 'profiles', 'roofline_traffic.json')
    if os.path.exists(p):
        try:
            return json.load(open(p)).get('rgcn_gather_bytes_per_launch')
        except Exception:
            return None
    return None


# ------------------------------------------------------------------------------------------------------
def cpu_reference_sample(tkg, torch, steps, warmup):
    """The reference's CPU path for the aggregate: its own op sequence per layer (RGCN.py:79-94:
    index_select of the [E,400] weights, bmm over E*100 1x2.2x2 products, index_add reduce, norm, self-loop
    mm, relu) restated in oracle/restate.py, on all host cores.  One step = ONE direction x 2 layers of one
    batch (a bounded sample of the GPU arm's step, which is two directions)."""
    from oracle import restate
    from renet_b200 import utils
    q = _cpu_quota()
    # all the host threads the container can actually run: more threads than the cgroup quota only thrash
    torch.set_num_threads(max(1, min(os.cpu_count() or 1, int(q + 0.5))) if q else (os.cpu_count() or 1))
    q, sh, oh = tkg.batch(0, BATCH, tail_only=False)
    hb = utils.assemble_history_batch_host(sh[0], sh[1], q[:, 0], tkg.graph_dict)
    g = hb.graph
    N, E = len(g['node_ent']), len(g['col_src'])
    gen = torch.Generator().manual_seed(0)
    ent = torch.randn(tkg.num_e, H_DIM, generator=gen) * 0.1
    W = [torch.randn(2 * tkg.num_r, 4 * NUM_BASES, generator=gen) * 0.1 for _ in range(2)]
    Wl = [torch.randn(H_DIM, H_DIM, generator=gen) * 0.07 for _ in range(2)]
    src = torch.from_numpy(g['col_src'].astype(np.int64))
    dst = torch.from_numpy(np.repeat(np.arange(N), np.diff(g['row_ptr'])))
    et = torch.from_numpy(g['col_type_s'].astype(np.int64))
    norm = torch.from_numpy(g['norm'])
    ids = torch.from_numpy(g['node_ent'])

    def step():
        H0 = ent[ids]
        H1 = restate.rgcn_block_layer_ref_ops(H0, W[0], Wl[0], src, dst, et, norm, True, NUM_BASES)
        return restate.rgcn_block_layer_ref_ops(H1, W[1], Wl[1], src, dst, et, norm, False, NUM_BASES)

    with torch.no_grad():
        for _ in range(warmup):
            step()
        times = []
        for _ in range(steps):
            t0 = time.perf_counter()
            step()
            times.append(time.perf_counter() - t0)
    med = float(np.median(times))
    return {'value': 2 * E / med, 'unit': UNIT, 'cores': torch.get_num_threads(), 'host_cpu_quota': _cpu_quota(), 'kind': 'port',
            'sample': 'one direction x 2 layers of one batch (N=%d, E=%d), reference op sequence '
                      '(index_select+bmm+index_add) in torch CPU fp32, median of %d' % (N, E, steps),
            'ms_per_step': med * 1e3, 'edge_msgs_per_step': 2 * E}


def run_reference(args):
    """--impl reference: the reference's CPU implementation of the path on the host cores."""
    rank = int(os.environ.get('RANK', '0'))
    if rank != 0:
        return
    import torch
    from renet_b200 import synthetic
    tkg = synthetic.SyntheticTKG(WORKLOADS[args.workload][0] or 'icews18', seed=999, num_timestamps=args.timestamps, h_dim=H_DIM)
    steps = max(1, min(args.steps, 5))
    res = cpu_reference_sample(tkg, torch, steps, max(1, min(args.warmup, 1)))
    line = {'impl': 'reference', 'metric': METRIC, 'value': res['value'], 'unit': UNIT, 'n_gpus': args.gpus,
            'steps': steps, 'warmup': 1, 'ms_per_step': res['ms_per_step'], 'higher_is_better': True,
            'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
            'config': {'workload': WORKLOAD, 'sample': res['sample']},
            'cpu_baseline': {k: res[k] for k in ('value', 'unit', 'cores', 'host_cpu_quota', 'kind', 'sample')},
            'e2e': {'value': res['value'], 'unit': UNIT, 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0},
            'gpu_launches': 0}
    print(json.dumps(line))



# ------------------------------------------------------------------------------------------------------
def train_region(args, tkg, pool, global_emb, dev, world, torch, dist):
    """One reference training step per iteration (train.py:136-143) on this rank's shard of the global batch
    (1024 samples per rank, global batch 1024 x world): RENet.forward x2 directions -> backward through the CUDA
    backward kernels -> gradient all-reduce (NCCL, bucketed, launched from autograd hooks while backward still runs)
    -> clip_grad_norm_ -> Adam (csrc/optim.cu).  Device-timed over pre-built batches resident in HBM, rotating over the
    pool; the backward graph structures (CSR by source, relation-grouped edges) are rebuilt every step, as for a fresh
    batch.  Phase times come from CUDA events on the compute stream: `allreduce_exposed_ms` is the time that stream
    spends waiting for NCCL after the last backward kernel."""
    from renet_b200 import _lib
    from renet_b200.model import RENet
    from renet_b200.parallel import DataParallelTrainer
    torch.manual_seed(999)
    model = RENet(tkg.num_e, H_DIM, tkg.num_r, dropout=args.dropout).to(dev).train()
    model.global_emb = global_emb
    tr = DataParallelTrainer(model, lr=1e-3, weight_decay=1e-5, grad_norm=1.0, record_events=True)
    for e in pool:
        if 'q_dev' not in e:
            e['q_dev'] = torch.from_numpy(e['q']).to(dev)

    def one(e):
        for d in e['dirs']:
            d['hb'].graph._bwd = {}
        return tr.train_step(e['q_dev'], e['dirs'][0]['hb'], e['dirs'][1]['hb'], tkg.graph_dict)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    warm = max(3, args.warmup)
    for i in range(warm):
        one(pool[i % len(pool)])
    barrier()
    n0 = _lib.launch_count()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    evs, msgs, losses = [], 0, []
    for i in range(args.steps):
        e = pool[(warm + i) % len(pool)]
        losses.append(one(e))
        evs.append(tr.last_events)
        msgs += sum(2 * d['g'].E for d in e['dirs'])
    end.record()
    barrier()
    launches = _lib.launch_count() - n0
    ms = start.elapsed_time(end)
    phases = np.zeros(4)
    for ev in evs:
        phases += [ev[k].elapsed_time(ev[k + 1]) for k in range(4)]
    phases /= len(evs)
    t = torch.tensor([ms, float(msgs)] + list(phases), device=dev, dtype=torch.float64)
    exposed_min = float(phases[2])
    if world > 1:
        tmax = t.clone(); dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        tsum = t.clone(); dist.all_reduce(tsum, op=dist.ReduceOp.SUM)
        tmin = t.clone(); dist.all_reduce(tmin, op=dist.ReduceOp.MIN)
        ms, msgs = tmax[0].item(), tsum[1].item()
        phases = tmax[2:].cpu().numpy()
        exposed_min = tmin[4].item()
    loss = float(torch.stack(losses).mean())
    tr.close()
    return {'value': msgs / (ms * 1e-3), 'unit': UNIT, 'ms_per_step': ms / args.steps, 'steps': args.steps, 'warmup': warm,
            'forward_ms': float(phases[0]), 'backward_ms': float(phases[1]), 'allreduce_exposed_ms': float(phases[2]),
            'optimizer_ms': float(phases[3]), 'allreduce_exposed_min_over_ranks_ms': exposed_min,
            'note': 'phase times are CUDA-event spans on the compute stream, max over ranks; the exposed all-reduce of the slowest-'
                    'waiting rank includes the time it waits for the LAST rank to reach the collective (rank skew), the min over '
                    'ranks is the communication that no rank could hide',
            'global_batch': BATCH * world, 'dropout': args.dropout,
            'grad_bytes_allreduced_per_step': int(tr.total * 4) if world > 1 else 0, 'buckets': len(tr.buckets),
            'collective': ('nccl all_reduce(sum) of the flat fp32 gradient in %d buckets, launched from autograd hooks during '
                           'backward' % len(tr.buckets)) if world > 1 else 'none (1 GPU)',
            'gpu_launches': int(launches), 'mean_loss': loss,
            'what': 'train.py:136-143 per rank: RENet.forward x2 directions (RGCN x2 + fused read-out/GRU + decoder/CE) -> backward '
                    '-> gradient all-reduce -> clip_grad_norm_(1.0) -> Adam(lr 1e-3, wd 1e-5); phase times are max over ranks'}


DUMP_SAMPLE_ROWS = 8192


def dump_outputs(out_dir, e, np):
    """The arrays one timed step hands its caller, for both directions: `h2_<dir>` = layer-2 output (the read-out rows that
    feed the GRU, [S, 200]) in full, `h1_<dir>` = layer-1 output ([N, 200], 27 MB per direction at the ICEWS18 shape) on a
    fixed seeded sample of DUMP_SAMPLE_ROWS rows whose indices are `h1_<dir>_rows`.  float32; about 15 MB in all."""
    os.makedirs(out_dir, exist_ok=True)
    for d in e['dirs']:
        tag = 'obj' if d['reverse'] else 'subj'
        H1 = d['H1'].float().cpu().numpy()
        rows = np.sort(np.random.RandomState(0).choice(len(H1), min(len(H1), DUMP_SAMPLE_ROWS), replace=False))
        np.save(os.path.join(out_dir, 'h1_%s.npy' % tag), H1[rows])
        np.save(os.path.join(out_dir, 'h1_%s_rows.npy' % tag), rows.astype(np.float64))
        np.save(os.path.join(out_dir, 'h2_%s.npy' % tag), d['H2'].float().cpu().numpy())


# ------------------------------------------------------------------------------------------------------
def run_ours(args):
    import torch
    import torch.distributed as dist
    import torch.nn.functional as F
    from renet_b200 import _lib, synthetic, utils
    from renet_b200.model import RENet

    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    # before any worker thread exists: keep this rank (loader threads, OpenMP pool, consumer) on its GPU's NUMA node and
    # on its own share of the cores
    from renet_b200 import affinity
    pin = affinity.pin_rank(local, int(os.environ.get('LOCAL_WORLD_SIZE', world))) if world > 1 else {'pinned': False, 'why': '1 rank'}
    if not torch.cuda.is_available():
        raise SystemExit('bench.py: no CUDA device -- the hot path has no CPU fallback')
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
    L = _lib.lib()

    # ---- workload: every rank owns its own shard of the stream (weak scaling, no data-path collective)
    tkg = synthetic.SyntheticTKG(WORKLOADS[args.workload][0], seed=999 + rank, num_timestamps=args.timestamps, h_dim=H_DIM)
    torch.manual_seed(999)
    model = RENet(tkg.num_e, H_DIM, tkg.num_r, dropout=0).to(dev).eval()
    model.global_emb = {t: v.to(dev) for t, v in tkg.global_emb.items()}
    agg = model.aggregator
    ent = model.ent_embeds.detach()
    R2 = 2 * tkg.num_r

    from renet_b200 import hoststore
    if args.host_batcher:
        hoststore.DEVICE_EDGES = False
    gstore = hoststore.GraphStore(tkg.graph_dict)
    hs_s = hoststore.HistoryStore(tkg.s_hist, tkg.s_hist_t, tkg.quads[:, 0], gstore, reverse=False)
    hs_o = hoststore.HistoryStore(tkg.o_hist, tkg.o_hist_t, tkg.quads[:, 2], gstore, reverse=True)
    pool = []
    for i in range(args.pool):
        q, sh, oh = tkg.batch(i, BATCH, tail_only=False)
        sel = tkg.batch_indices(i, BATCH, tail_only=False)
        entry = {'q': q, 'sh': sh, 'oh': oh, 'dirs': [], 'vs': hs_s.select(sel), 'vo': hs_o.select(sel)}
        for hist, col, reverse in ((sh, 0, False), (oh, 2, True)):
            hb = utils.assemble_history_batch(hist[0], hist[1], q[:, col], tkg.graph_dict, dev)
            g = hb.graph
            # layer 2 runs on the read-out sub-graph (Aggregator.py:140 keeps only the read-out rows of its output; SURVEY.md
            # section 8(a) optimisation (i)); like the CSR itself it is graph preprocessing, built by the batcher
            sub = g.readout_sub(hb.readout, reverse)
            entry['dirs'].append({'hb': hb, 'g': g, 'reverse': reverse, 'ct': g.col_type(reverse), 'sub': sub,
                                  'H1': torch.empty(g.N, H_DIM, device=dev), 'H2': torch.empty(hb.S, H_DIM, device=dev)})
        pool.append(entry)
    # The synthetic stream is millions of small Python objects (history lists of numpy arrays, per-timestamp graphs): a full
    # garbage collection that lands inside a timed region stalls the launching thread for up to a second (seen once per run
    # in the event-timed region of the GDELT workload: one 1.1 s "launch").  Everything built so far is permanent: take it
    # out of the collector's sight.
    import gc
    gc.collect()
    gc.freeze()
    msgs_per_step = [sum(2 * d['g'].E for d in e['dirs']) for e in pool]              # over the FULL E, as SURVEY 8(a) demands
    msgs_executed = [sum(d['g'].E + d['sub'].E for d in e['dirs']) for e in pool]     # edges the kernels actually walk
    pool_bytes = sum(sum(d['g'].E * 12 + d['g'].N * (8 + 1600) for d in e['dirs']) for e in pool)
    if args.mode == 'train':
        clocks = ClockSampler(local)
        clocks.start()
        train = train_region(args, tkg, pool, model.global_emb, dev, world, torch, dist)
        clk = clocks.stop()
        if rank == 0:
            print(json.dumps({'metric': 'training_step_edge_messages_per_sec', 'value': train['value'], 'unit': UNIT, 'n_gpus': world,
                              'steps': args.steps, 'warmup': train['warmup'], 'ms_per_step': train['ms_per_step'],
                              'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
                              'config': {'workload': WORKLOAD, 'global_batch': BATCH * world, 'l2': 'rotating-pool',
                                         'pool_batches': len(pool), 'parallelism': 'dp%d (replicated parameters, NCCL gradient all-reduce)' % world},
                              'clocks': clk, 'gpu_launches': train['gpu_launches'], 'train': train}))
        if world > 1:
            dist.destroy_process_group()
        return
    W1, L1, W2, L2 = (agg.rgcn1.weight.detach(), agg.rgcn1.loop_weight.detach(), agg.rgcn2.weight.detach(),
                      agg.rgcn2.loop_weight.detach())
    P = _lib.ptr
    stream = _lib.stream()
    hot_rel = gstore.hot_relations(dev)

    def layer(d, H, h_index, W, Wl, out, relu, ev=None, sub=None):
        g = d['g']
        if sub is None:
            rows, loop_index, rp, cs, ct, nm, n_e = g.N, h_index, g.row_ptr, g.col_src, d['ct'], g.norm, g.E
        else:       # read-out sub-graph: S compact destinations, sources = rows of H
            rows, loop_index, rp, cs, ct, nm, n_e = sub.N, sub.uniq, sub.row_ptr, sub.col_src, sub.col_type(d['reverse']), sub.norm, sub.E_cap
        if ev is not None:
            ev[2].record()
        _lib.check(L.renet_selfloop_gemm(P(H), P(loop_index), P(Wl), P(out), rows, H_DIM, H_DIM, stream), 'gemm')
        if ev is not None:
            ev[0].record()
        hot = hot_rel[d['reverse']]     # the dataset's relation ranking (GraphStore.hot_relations): part of the graph store
        _lib.check(L.renet_rgcn_gather_hot(P(H), P(h_index), P(W), P(rp), P(cs), P(ct), P(nm), P(out), rows, n_e, H_DIM, H_DIM,
                                           NUM_BASES, R2, int(relu), 1, P(hot), hot.numel(), stream), 'gather')
        if ev is not None:
            ev[1].record()

    step_no = [0]

    def device_step(e, events=None):
        # every step is a new weight generation, as in training (the optimiser changes the weights between steps): the
        # tensor-core engine packs each self-loop matrix once per step and both directions use the image
        step_no[0] += 1
        L.renet_set_weight_generation(step_no[0])
        k = 0
        for d in e['dirs']:
            layer(d, ent, d['g'].node_ent, W1, L1, d['H1'], True, events[k] if events else None)
            layer(d, d['H1'], None, W2, L2, d['H2'], False, events[k + 1] if events else None, sub=d['sub'])
            k += 2
        L.renet_set_weight_generation(-1)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- region A: `value` ----------------------------------------------------------------------------
    for i in range(args.warmup):
        device_step(pool[i % len(pool)])
    clocks = ClockSampler(local)
    barrier()
    clocks.start()
    n0 = _lib.launch_count()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    total_msgs = 0
    for i in range(args.steps):
        device_step(pool[(args.warmup + i) % len(pool)])
        total_msgs += msgs_per_step[(args.warmup + i) % len(pool)]
    end.record()
    barrier()
    launches = _lib.launch_count() - n0
    elapsed_ms = start.elapsed_time(end)
    clk = clocks.stop()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, pool[(args.warmup + args.steps - 1) % len(pool)], np)
    t = torch.tensor([elapsed_ms, float(total_msgs)], device=dev, dtype=torch.float64)
    if world > 1:
        tmax = t.clone(); dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        tsum = t.clone(); dist.all_reduce(tsum, op=dist.ReduceOp.SUM)
        elapsed_ms, total_msgs = tmax[0].item(), tsum[1].item()
    value = total_msgs / (elapsed_ms * 1e-3)

    # ---- region B: per-launch time of the fused gather kernel (roofline) ---------------------------------
    ev_steps = []
    for i in range(args.steps):
        evs = [tuple(torch.cuda.Event(enable_timing=True) for _ in range(3)) for _ in range(4)]
        device_step(pool[(args.warmup + i) % len(pool)], evs)
        ev_steps.append((pool[(args.warmup + i) % len(pool)], evs))
    torch.cuda.synchronize()
    g_ms, g_bytes, g2_ms, g2_bytes, mm_ms, mm_bytes, mm_flops = [], [], [], [], [], [], []
    for e, evs in ev_steps:
        for k, (a, b, c) in enumerate(evs):
            d = e['dirs'][k // 2]
            if k % 2 == 0:        # layer 1: the whole batched graph
                g_ms.append(a.elapsed_time(b))
                g_bytes.append(algorithmic_bytes(d['g'].N, d['g'].E, R2))
                # self-loop GEMM of the same layer: gathered input rows + output rows + the weight matrix
                mm_ms.append(c.elapsed_time(a))
                mm_bytes.append(d['g'].N * (H_DIM * 4 * 2 + 4) + H_DIM * H_DIM * 4)
                mm_flops.append(2.0 * d['g'].N * H_DIM * H_DIM)
            else:                 # layer 2: the read-out sub-graph (U destinations, E2 edges)
                g2_ms.append(a.elapsed_time(b))
                g2_bytes.append(algorithmic_bytes(d['sub'].sizes()[0], d['sub'].E, R2))
    peak, peak_src = measured_peak_gbs()
    achieved = float(np.sum(g_bytes) / (np.sum(g_ms) * 1e-3) / 1e9)
    roofline = {'kernel': 'rgcn_gather_stream_kernel', 'bound': 'hbm', 'achieved': achieved, 'peak': peak,
                'unit': 'GB/s', 'frac': achieved / peak, 'traffic': ncu_traffic(), 'peak_source': peak_src,
                'avg_launch_us': float(np.mean(g_ms) * 1e3), 'algorithmic_bytes_per_launch': float(np.mean(g_bytes)),
                'launches': 'layer-1 launches (whole batched graph); layer 2 runs the same kernel on the read-out sub-graph: '
                            '%.1f us per launch, %.0f GB/s of its own algorithmic bytes' % (float(np.mean(g2_ms) * 1e3), float(np.sum(g2_bytes) / (np.sum(g2_ms) * 1e-3) / 1e9)),
                'note': 'features are L2-resident at this size (25 MB); DRAM traffic is below the algorithmic bytes'}

    mm_achieved = float(np.sum(mm_bytes) / (np.sum(mm_ms) * 1e-3) / 1e9)
    tf32_peak, tf32_src = measured_peak_tf32()
    roofline_gemm = {'kernel': 'umma_gemm_packed_kernel (layer-1 self-loop product, wgmma 3xTF32)', 'bound': 'hbm',
                     'achieved': mm_achieved, 'peak': peak, 'unit': 'GB/s', 'frac': mm_achieved / peak,
                     'avg_launch_us': float(np.mean(mm_ms) * 1e3), 'algorithmic_bytes_per_launch': float(np.mean(mm_bytes)),
                     'tensor_tflops_3xtf32': float(3 * np.sum(mm_flops) / (np.sum(mm_ms) * 1e-3) / 1e12), 'tf32_peak_tflops': tf32_peak,
                     'note': 'N x 200 x 200 per launch: the memory floor (rows in + rows out) and the 3xTF32 tensor floor are within '
                             '20 % of each other; timed with the packing launch of a new weight generation included'}

    if os.environ.get('RENET_STREAM_TL') == '1' and rank == 0:
        # debug: per-warp time stamps of ONE layer-1 gather launch in the middle of a step (tools/stream_timeline.py explains them)
        WARPS = int(os.environ.get('RENET_STREAM_WARPS', '32'))
        buf = torch.zeros(132 * WARPS * 8, dtype=torch.int64, device=dev)
        e = pool[(args.warmup + 3) % len(pool)]
        d = e['dirs'][0]
        _lib.check(L.renet_selfloop_gemm(P(ent), P(d['g'].node_ent), P(L1), P(d['H1']), d['g'].N, H_DIM, H_DIM, stream), 'gemm')
        L.renet_debug_stream_timing(P(buf))
        hot = hot_rel[False]
        _lib.check(L.renet_rgcn_gather_hot(P(ent), P(d['g'].node_ent), P(W1), P(d['g'].row_ptr), P(d['g'].col_src), P(d['ct']), P(d['g'].norm),
                                           P(d['H1']), d['g'].N, d['g'].E, H_DIM, H_DIM, NUM_BASES, R2, 1, 1, P(hot), hot.numel(), stream), 'gather')
        torch.cuda.synchronize()
        L.renet_debug_stream_timing(None)
        t = buf.cpu().numpy().reshape(132, WARPS, 8).astype(np.float64)
        g0 = t[:, :, 5].min()
        ph = [(t[:, :, 1] - t[:, :, 0]) / 1980.0, (t[:, :, 2] - t[:, :, 1]) / 1980.0, (t[:, :, 3] - t[:, :, 2]) / 1980.0, (t[:, :, 4] - t[:, :, 3]) / 1980.0]
        sys.stderr.write('stream timeline in context: span %.1f us, entry skew %.1f us; medians (us): search %.1f, prologue %.1f, loop %.1f, tail %.1f; '
                         'max loop %.1f\n' % ((t[:, :, 6].max() - g0) / 1e3, (t[:, :, 5].min(1).max() - g0) / 1e3, np.median(ph[0]), np.median(ph[1]),
                                              np.median(ph[2]), np.median(ph[3]), ph[2].max()))

    # ---- GRU (reported separately) -------------------------------------------------------------------------
    from renet_b200.gru import fused_gru
    gru_ms, roofline_gru = None, None
    try:
        with torch.no_grad():
            e = pool[0]
            rel = model.rel_embeds[:tkg.num_r]
            d = e['dirs'][0]
            hb = d['hb']
            seq = agg._sorted_ids(hb, torch.from_numpy(e['q'][:, 0]).to(dev), torch.from_numpy(e['q'][:, 1]).to(dev), dev)
            glob = utils.global_rows(model.global_emb, hb.times, H_DIM, dev)
            for _ in range(2):
                fused_gru(d['H2'], ent, rel, glob, hb, seq[2], seq[3], model.encoder, model.encoder_r, readout=d['sub'].readout_c)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(5):
                fused_gru(d['H2'], ent, rel, glob, hb, seq[2], seq[3], model.encoder, model.encoder_r, readout=d['sub'].readout_c)
            b.record(); torch.cuda.synchronize()
            gru_ms = a.elapsed_time(b) / 5
            S_rows, Q_seq = int(hb.S), int(len(hb.seq_len))
            steps_rows = int(np.sum(hb.seq_len))                       # sum over time steps of the active sequences
            flops = 2.0 * H_DIM * 6 * H_DIM * (S_rows + 2 * Q_seq + len(hb.times) + steps_rows)
            roofline_gru = {'kernel': 'fused read-out + GRU of one direction: 4 wgmma projection GEMMs + gru_recur_kernel (both encoders)',
                            'bound': 'tensor', 'achieved': 3 * flops / (gru_ms * 1e-3) / 1e12, 'peak': tf32_peak, 'unit': 'TFLOP/s',
                            'frac': 3 * flops / (gru_ms * 1e-3) / 1e12 / tf32_peak, 'peak_source': tf32_src, 'ms': gru_ms,
                            'algorithmic_flops': flops, 'rows': S_rows, 'sequences': Q_seq,
                            'note': 'achieved counts the 3 TF32 products per fp32 multiply-add that the 1e-4 parity bar costs; the '
                                    'recurrence is a chain of <= 10 dependent steps, i.e. latency-bound far below the tensor peak'}
    except Exception as ex:   # the aggregate metric does not depend on it
        gru_ms = 'failed: %s' % ex

    # ---- e2e: public API from host inputs ----------------------------------------------------------------------
    e2e = None
    if not args.no_e2e:
        def api_step(e, hbs, out_pinned):
            batch = e['q_pinned'].to(dev, non_blocking=True)                # triplets: pinned host -> device, every step
            outs, h2d = [], batch.numel() * 8 + sum(hb.h2d_bytes for hb in hbs)
            with torch.no_grad():
                for subj in (True, False):
                    s, r, o, s_h, s_q, _ = model.encode(batch, hbs[0], hbs[1], gstore, subject=subj)
                    outs.append(torch.cat((s_h, s_q), 1))
            res = torch.cat(outs)
            done = torch.cuda.Event()
            done.record()
            with torch.cuda.stream(copy_stream):                         # D2H of this step's GRU outputs on its own
                copy_stream.wait_event(done)                             # stream: overlaps the next step's kernels
                out_pinned[:res.shape[0]].copy_(res, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(copy_stream)
            res.record_stream(copy_stream)
            return h2d, res.numel() * 4, ev

        out_ring = [torch.empty(2 * BATCH, 2 * H_DIM).pin_memory() for _ in range(2)]
        copy_stream = torch.cuda.Stream(device=dev)
        for e in pool:
            e['q_pinned'] = torch.from_numpy(e['q']).pin_memory()

        def run_e2e(n_warm, n_steps, first):
            """ONE continuous stream of n_warm + n_steps steps through the loader; the clock starts when warm-up step
            n_warm-1 has completed on the GPU, with the loader in steady state (it stays `depth` steps ahead of the
            consumer at the start and at the end of the timed region alike), and stops when the last step's outputs are
            on the host."""
            entries = [pool[(first + i) % len(pool)] for i in range(n_warm + n_steps)]
            groups = ((e['vs'], e['vo']) for e in entries)
            h2d = d2h = 0
            prev = None
            checksum = 0.0
            graphs = []
            t0 = None
            # host inputs -> batch planning in worker threads (steps i+1, i+2 are prepared while step i runs on the GPU);
            # step i's result is read on the host (pinned D2H + event) right after step i+1 has been enqueued
            for i, (e, hbs) in enumerate(zip(entries, hoststore.prefetch(groups, dev, depth=E2E_DEPTH, workers=E2E_WORKERS))):
                if i == n_warm:
                    if prev is not None:
                        prev[0].synchronize()
                        checksum += float(prev[1][0, 0])
                        prev = None
                    barrier()
                    t0 = time.perf_counter()
                a, b, ev = api_step(e, hbs, out_ring[i & 1])
                if i >= n_warm:
                    h2d += a; d2h += b
                    # edge counts come back asynchronously and are summed after the loop; only the tiny handles are kept,
                    # so every batch's device memory returns to the allocator when its step is done
                    graphs.extend(hb.graph.edge_count_handle() for hb in hbs)
                if prev is not None:
                    prev[0].synchronize()
                    checksum += float(prev[1][0, 0])
                prev = (ev, out_ring[i & 1])
            if prev is not None:
                prev[0].synchronize()
                checksum += float(prev[1][0, 0])
            barrier()
            dt = time.perf_counter() - t0
            msgs = sum(2 * g.value() for g in graphs)
            return h2d, d2h, msgs, dt

        # loader threads per rank: 8 when the host has room; under a cgroup CPU quota leave a core per rank for the
        # consumer thread (a plan takes ~0.6 ms of one core, a step needs two: 2 threads keep up with a 1.3 ms step)
        quota = _cpu_quota()
        E2E_DEPTH = 4
        hoststore.reserve_pinned(4 * (E2E_DEPTH + 3))     # every staging buffer the loader can need, pinned up front
        E2E_WORKERS = max(2, min(8, _rank_cpu_budget() - int(os.environ.get('OMP_NUM_THREADS', '1')) - 1))
        k_e2e = args.steps
        # one full rotation over the pool of batches: the loader, the pinned pool and the caching allocator (whose block
        # sizes depend on the batch) have reached steady state before the clock starts
        w_e2e = max(len(pool) + 1, args.warmup)
        if os.environ.get('RENET_E2E_PROFILE') == '1' and rank == 0:      # debug: where the consumer thread's time goes
            import cProfile, pstats, io
            run_e2e(w_e2e, 20, 0)
            pr = cProfile.Profile()
            pr.enable()
            run_e2e(2, 100, 0)
            pr.disable()
            for key in ('tottime', 'cumulative'):
                buf = io.StringIO()
                pstats.Stats(pr, stream=buf).sort_stats(key).print_stats(28)
                sys.stderr.write(buf.getvalue())
        h2d, d2h, msgs, dt = run_e2e(w_e2e, k_e2e, 0)
        tt = torch.tensor([dt, float(msgs)], device=dev, dtype=torch.float64)
        if world > 1:
            a = tt.clone(); dist.all_reduce(a, op=dist.ReduceOp.MAX)
            b = tt.clone(); dist.all_reduce(b, op=dist.ReduceOp.SUM)
            dt, msgs = a[0].item(), b[1].item()
        e2e = {'value': msgs / dt, 'unit': UNIT, 'h2d_bytes_per_step': int(h2d / k_e2e), 'd2h_bytes_per_step': int(d2h / k_e2e),
               'ms_per_step': dt / k_e2e * 1e3, 'steps': k_e2e, 'warmup': w_e2e, 'cpu_pinning': pin,
               'host_threads': {'loader': E2E_WORKERS, 'omp': int(os.environ.get('OMP_NUM_THREADS', '0') or 0), 'rank_cpu_budget': _rank_cpu_budget()},
               'batcher': 'device (renet_host_plan_batch + renet_induce_edges)' if hoststore.DEVICE_EDGES else
                          'host (renet_host_assemble_batch)',
               'what': 'RENet.encode x2 directions from HOST inputs (flat history store + triplets; the per-timestamp graph '
                       'store is resident in HBM like the parameters): host planning of the batch (sample order, components, '
                       'node numbering, read-out rows; prepared %d steps ahead by %d worker threads)' % (E2E_DEPTH, E2E_WORKERS) + '  + one pinned H2D per '
                       'direction + induced-edge CSR build on the GPU + RGCN x2 + fused read-out/GRU + pinned D2H of the '
                       '[B,2h] outputs every step (read one step behind the enqueue front)'}

    train = None
    if not args.no_train:
        try:
            train = train_region(args, tkg, pool, model.global_emb, dev, world, torch, dist)
        except Exception as ex:          # the aggregate metric does not depend on it; a failure is reported, not hidden
            import traceback
            train = {'failed': '%s: %s' % (type(ex).__name__, ex), 'trace': traceback.format_exc()[-1500:]}

    cpu = None
    if rank == 0 and args.gpus == 1 and not args.no_cpu_baseline:
        cpu = cpu_reference_sample(tkg, torch, 3, 1)
        cpu = {k: cpu[k] for k in ('value', 'unit', 'cores', 'host_cpu_quota', 'kind', 'sample')}

    if rank == 0:
        g0 = pool[0]['dirs']
        line = {'metric': METRIC, 'value': value, 'unit': UNIT, 'n_gpus': world, 'steps': args.steps, 'warmup': args.warmup,
                'ms_per_step': elapsed_ms / args.steps, 'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None,
                'dtype': 'f32', 'data': 'synthetic',
                'config': {'workload': WORKLOAD, 'step': '2 directions x 2 RGCN layers (wgmma 3xTF32 self-loop GEMM + fused gather; layer 2 on the read-out sub-graph); every step is a new weight generation: each self-loop matrix is packed once per step and shared by both directions',
                           'nodes_per_direction': [d['g'].N for d in g0], 'edges_per_direction': [d['g'].E for d in g0],
                           'edge_msgs_per_step': msgs_per_step[0], 'edge_msgs_executed_per_step': msgs_executed[0],
                           'layer2': 'read-out sub-graph only (identical on every consumed row, Aggregator.py:140); value counts the full E for both layers',
                           'l2': 'rotating-pool', 'pool_batches': len(pool),
                           'pool_bytes': int(pool_bytes), 'parallelism': 'dp%d (independent shards, no data-path collective)' % world},
                'clocks': clk, 'e2e': e2e, 'gpu_launches': int(launches), 'roofline': roofline, 'cpu_baseline': cpu,
                'gru_ms_one_direction': gru_ms, 'roofline_gemm': roofline_gemm, 'roofline_gru': roofline_gru, 'train': train}
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    a = parse()
    if a.timestamps is None:
        a.timestamps = WORKLOADS[a.workload][1]
    WORKLOAD = WORKLOADS[a.workload][2]
    if a.dump_outputs and (a.workload == 'synth1m' or a.impl == 'reference'):
        raise SystemExit('bench.py: --dump-outputs covers the CUDA arm of the icews18 and gdelt workloads')
    if a.workload == 'synth1m' and a.impl != 'reference':
        from bench_synth import run_synth1m
        run_synth1m(a, WORKLOAD, METRIC, UNIT, ClockSampler, measured_peak_gbs)
    elif a.impl == 'reference':
        run_reference(a)
    else:
        run_ours(a)
