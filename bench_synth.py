"""bench.py --workload synth1m: BASELINE.json configs[4] -- a synthetic TKG shard of 1M entities / 500 relations / 250
timesteps per GPU with mean in-degree 32 (N = 1M nodes, E = 32M directed edges per GPU, weak scaling over GPUs).  The only
configuration whose feature matrix (800 MB) does not fit the 50 MB L2, i.e. where HBM is the true bound of the gather.
Aggregate + GRU only (SURVEY.md section 8(d): the 1M-class decoder is out of scope).

A step = one direction over the shard's batched graph: layer 1 (self-loop GEMM + fused gather over all N / E), layer 2
on the read-out sub-graph, fused read-out + both GRUs over Q = 32768 sequences of length 10.
"""
import json
import os
import time

import numpy as np

H_DIM, NUM_BASES = 200, 100


def make_shard(torch, N, G, R, Q, seq_len, seed, device):
    """Edge list (both directions, reference utils.get_big_graph order: [s->o.., o->s..] with types (r, r+R)), read-out rows
    and sequence bookkeeping of one shard, generated on ``device`` with torch's generator."""
    g = torch.Generator(device=device).manual_seed(seed)
    size = N // G
    half = 16 * N                                   # undirected events; E = 2 * half directed edges, mean in-degree 32
    comp = torch.randint(0, G, (half,), generator=g, device=device)
    # endpoint skew inside a component: u^2.5 concentrates on the first rows (hubs), like the Zipf endpoint skew of the real sets
    a = (torch.rand(half, generator=g, device=device) ** 2.5 * size).long().clamp_(max=size - 1)
    b = (torch.rand(half, generator=g, device=device) ** 1.5 * size).long().clamp_(max=size - 1)
    s, o = comp * size + a, comp * size + b
    r = (torch.rand(half, generator=g, device=device) ** 3.0 * R).long().clamp_(max=R - 1)
    src = torch.cat((s, o)).to(torch.int32)
    dst = torch.cat((o, s)).to(torch.int32)
    type_s = torch.cat((r, r + R)).to(torch.int32)
    # read-out rows: sequence q at step t reads a hub-biased node of component (q + t) % G
    qi = torch.arange(Q, device=device).repeat_interleave(seq_len)
    ti = torch.arange(seq_len, device=device).repeat(Q)
    rc = (qi + ti) % G
    rn = (torch.rand(Q * seq_len, generator=g, device=device) ** 2.5 * size).long().clamp_(max=size - 1)
    readout = (rc * size + rn).to(torch.int32)
    return dict(src=src, dst=dst, type_s=type_s, readout=readout, row_glob=rc.to(torch.int32), seq_s=readout[::seq_len].clone())


def run_synth1m(args, WORKLOAD, METRIC, UNIT, ClockSampler, measured_peak_gbs):
    import torch
    import torch.distributed as dist
    from renet_b200 import _lib
    from renet_b200.graph import ReadoutSubgraph, build_csr
    from renet_b200.model import RENet
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if not torch.cuda.is_available():
        raise SystemExit('bench.py: no CUDA device -- the hot path has no CPU fallback')
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
    L, P = _lib.lib(), _lib.ptr
    N, G, R, Q, SL = int(args.synth_nodes), 250, 500, 32768, 10
    R2 = 2 * R
    sh = make_shard(torch, N, G, R, Q, SL, 999 + rank, dev)
    E = int(sh['src'].numel())
    import gc
    gc.collect()
    gc.freeze()          # nothing built so far is garbage: keep full collections out of the timed regions
    S = Q * SL
    # ---- graph preprocessing (not timed): CSR by destination, norm, read-out sub-graph
    row_ptr, col_src, col_type, _ = build_csr(sh['dst'], sh['src'], sh['type_s'], N)
    deg = (row_ptr[1:] - row_ptr[:-1]).float().clamp_(min=1)
    norm = 1.0 / deg

    class _G:      # the surface ReadoutSubgraph reads
        pass
    g = _G()
    g.device, g.N, g.row_ptr, g.col_src, g.norm = dev, N, row_ptr, col_src, norm
    g.col_type = lambda reverse: col_type
    g.hot_rel = lambda reverse: None
    sub = ReadoutSubgraph(g, sh['readout'], False)
    U, E2 = sub.sizes()
    torch.manual_seed(999)
    ent = torch.randn(N, H_DIM, device=dev) * 0.1                       # ent_embeds: 1M x 200 (800 MB); node i <-> entity perm[i]
    node_ent = torch.randperm(N, device=dev).to(torch.int32)
    m = RENet(1024, H_DIM, R, dropout=0).to(dev).eval()                 # only its RGCN / GRU parameters are used
    W1, L1, W2, L2 = (m.aggregator.rgcn1.weight.detach(), m.aggregator.rgcn1.loop_weight.detach(),
                      m.aggregator.rgcn2.weight.detach(), m.aggregator.rgcn2.loop_weight.detach())
    rel = torch.randn(R, H_DIM, device=dev) * 0.1
    glob = torch.randn(G, H_DIM, device=dev) * 0.1
    seq_r = torch.randint(0, R, (Q,), device=dev, dtype=torch.int32)
    seq_len = torch.full((Q,), SL, dtype=torch.int32, device=dev)
    seq_start = (torch.arange(Q, device=dev) * SL).to(torch.int32)
    bs = np.full(SL, Q, dtype=np.int32)
    H1 = torch.empty(N, H_DIM, device=dev)
    H2 = torch.empty(S, H_DIM, device=dev)
    hn = torch.zeros(2, Q, H_DIM, device=dev)
    nbytes = int(L.renet_gru_workspace_bytes(S, Q, G, H_DIM))
    ws = torch.empty(nbytes // 4 + 4, dtype=torch.float32, device=dev)
    from renet_b200.gru import _gru_params
    p4, p3 = _gru_params(m.encoder), _gru_params(m.encoder_r)
    stream = _lib.stream()

    def step(ev=None):
        _lib.check(L.renet_selfloop_gemm(P(ent), P(node_ent), P(L1), P(H1), N, H_DIM, H_DIM, stream), 'gemm1')
        if ev:
            ev[0].record()
        _lib.check(L.renet_rgcn_gather(P(ent), P(node_ent), P(W1), P(row_ptr), P(col_src), P(col_type), P(norm), P(H1), N, E,
                                       H_DIM, H_DIM, NUM_BASES, R2, 1, 1, stream), 'gather1')
        if ev:
            ev[1].record()
        _lib.check(L.renet_selfloop_gemm(P(H1), P(sub.uniq), P(L2), P(H2), S, H_DIM, H_DIM, stream), 'gemm2')
        _lib.check(L.renet_rgcn_gather(P(H1), None, P(W2), P(sub.row_ptr), P(sub.col_src), P(sub.col_type(False)), P(sub.norm),
                                       P(H2), S, sub.E_cap, H_DIM, H_DIM, NUM_BASES, R2, 0, 1, stream), 'gather2')
        if ev:
            ev[2].record()
        rc = L.renet_gru_fwd(P(H2), P(sub.readout_c), P(sh['row_glob']), P(glob), P(ent), P(rel), P(sh['seq_s']), P(seq_r),
                             P(seq_len), P(seq_start), bs.ctypes.data_as(_lib.ctypes.c_void_p), SL, P(p4[0]), P(p4[1]), P(p4[2]),
                             P(p4[3]), P(p3[0]), P(p3[1]), P(p3[2]), P(p3[3]), P(hn[0]), P(hn[1]), S, Q, G, H_DIM, P(ws), nbytes,
                             stream)
        _lib.check(rc, 'gru')
        if ev:
            ev[3].record()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for _ in range(max(3, args.warmup)):
        step()
    clocks = ClockSampler(local)
    barrier()
    clocks.start()
    n0 = _lib.launch_count()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.steps):
        step()
    b.record()
    barrier()
    launches = _lib.launch_count() - n0
    ms = a.elapsed_time(b)
    clk = clocks.stop()
    # per-kernel split (second region, events between launches)
    evs = []
    for _ in range(min(args.steps, 10)):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        e[4].record()
        step(e[:4])
        evs.append(e)
    torch.cuda.synchronize()
    gemm1 = float(np.mean([e[4].elapsed_time(e[0]) for e in evs]))
    gath1 = float(np.mean([e[0].elapsed_time(e[1]) for e in evs]))
    lay2 = float(np.mean([e[1].elapsed_time(e[2]) for e in evs]))
    gru = float(np.mean([e[2].elapsed_time(e[3]) for e in evs]))
    msgs = 2.0 * E * args.steps                                          # both layers over the FULL E (SURVEY 8(a))
    t = torch.tensor([ms, msgs], device=dev, dtype=torch.float64)
    if world > 1:
        tmax = t.clone(); dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        tsum = t.clone(); dist.all_reduce(tsum, op=dist.ReduceOp.SUM)
        ms, msgs = tmax[0].item(), tsum[1].item()
    peak, peak_src = measured_peak_gbs()
    alg = E * (4 * H_DIM + 12) + N * (8 * H_DIM + 4) + R2 * (H_DIM * H_DIM // NUM_BASES) * 4
    achieved = alg / (gath1 * 1e-3) / 1e9
    traffic = None
    tp = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'profiles', 'roofline_traffic_synth1m.json')
    if os.path.exists(tp):
        try:
            traffic = json.load(open(tp)).get('rgcn_gather_bytes_per_launch')
        except Exception:
            traffic = None
    # ---- e2e: the same step from HOST inputs: pinned COO edge list + read-out rows -> H2D -> CSR build + norm + read-out
    # sub-graph on the GPU -> the step -> D2H of the GRU states
    pin = {k: sh[k].cpu().pin_memory() for k in ('src', 'dst', 'type_s', 'readout')}
    out_pinned = torch.empty(2, Q, H_DIM).pin_memory()

    def e2e_step():
        nonlocal row_ptr, col_src, col_type, norm, sub
        d = {k: v.to(dev, non_blocking=True) for k, v in pin.items()}
        row_ptr, col_src, col_type, _ = build_csr(d['dst'], d['src'], d['type_s'], N)
        norm = 1.0 / (row_ptr[1:] - row_ptr[:-1]).float().clamp_(min=1)
        g.row_ptr, g.col_src, g.norm = row_ptr, col_src, norm
        sub = ReadoutSubgraph(g, d['readout'], False)
        step()
        out_pinned.copy_(hn, non_blocking=True)
        torch.cuda.synchronize()
        return sum(v.numel() * v.element_size() for v in pin.values()), out_pinned.numel() * 4
    e2e_step()
    barrier()
    t0 = time.perf_counter()
    k_e2e = max(3, min(args.steps, 5))
    for _ in range(k_e2e):
        h2d, d2h = e2e_step()
    barrier()
    dt = time.perf_counter() - t0
    tt = torch.tensor([dt], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    e2e = {'value': 2.0 * E * k_e2e * world / tt.item(), 'unit': UNIT, 'h2d_bytes_per_step': int(h2d), 'd2h_bytes_per_step': int(d2h),
           'ms_per_step': tt.item() / k_e2e * 1e3, 'steps': k_e2e,
           'what': 'pinned host COO edge list (src, dst, type) + read-out rows -> H2D -> CSR build (renet_build_csr) + norm + read-out '
                   'sub-graph on the GPU -> layer 1 + layer 2 + fused read-out/GRU -> pinned D2H of the GRU states, synchronous per step'}
    if rank == 0:
        print(json.dumps({
            'metric': METRIC, 'value': msgs / (ms * 1e-3), 'unit': UNIT, 'n_gpus': world, 'steps': args.steps,
            'warmup': max(3, args.warmup), 'ms_per_step': ms / args.steps, 'higher_is_better': True, 'scaling': 'weak',
            'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
            'config': {'workload': WORKLOAD, 'nodes_per_gpu': N, 'edges_per_gpu': E, 'relations': R, 'components': G,
                       'readout_rows': S, 'sequences': Q, 'readout_nodes': U, 'readout_subgraph_edges': E2,
                       'step': 'one direction: layer 1 over the whole shard, layer 2 on the read-out sub-graph, fused read-out + GRUs',
                       'edge_msgs_per_step': 2 * E, 'edge_msgs_executed_per_step': E + E2,
                       'l2': 'inputs (800 MB of features + 384 MB of CSR per GPU) far exceed the 50 MB L2 of an H100',
                       'parallelism': 'dp%d (independent shards by timestep range, no data-path collective)' % world},
            'clocks': clk, 'e2e': e2e, 'gpu_launches': int(launches),
            'roofline': {'kernel': 'rgcn_gather_d200_kernel (layer 1, whole shard)', 'bound': 'hbm', 'achieved': achieved, 'peak': peak,
                         'unit': 'GB/s', 'frac': achieved / peak, 'traffic': traffic, 'peak_source': peak_src,
                         'avg_launch_us': gath1 * 1e3, 'algorithmic_bytes_per_launch': float(alg)},
            'split_ms': {'selfloop_gemm_layer1': gemm1, 'gather_layer1': gath1, 'layer2_readout_subgraph': lay2, 'readout_gru': gru},
            'cpu_baseline': None}))
    if world > 1:
        dist.destroy_process_group()
