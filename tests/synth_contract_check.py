"""Run in a subprocess by tests/test_gpu_synth_contract.py: the 1M-entity benchmark shard (bench.py --workload synth1m,
bench_synth.run_synth1m) per row against float64, forward and backward, at the shape bench.py measures.

The shard is bench_synth.make_shard with the bench's own arguments (N = --synth-nodes, G = 250, R = 500, Q = 32 768, length
10, seed 999) and the operands are drawn in the bench's order, so the five C calls of the bench's step() run here on the
same values and with the same arguments: the duck-typed parent graph for ReadoutSubgraph, sub.E_cap as layer 2's edge
count and renet_gru_workspace_bytes(S, Q, G, 200).

Every stage is checked from the kernel's own inputs to that stage, so errors do not compound and each bar stays tight, and
every row is compared.  The float64 restatements run in chunks of 2^19 edges (0.8 GB of messages per chunk), and layer 1
is restated and compared in blocks of 2^19 destinations, so that no [N, 200] float64 array but the chain's H1 is held
(the 4 M-node shard's forward peaks at ~ 30 GB instead of ~ 70 GB).
  1. layer-1 self-loop renet_selfloop_gemm(ent, node_ent, L1): per row within (K + 4) 2^-24 sum |a b| (K = 200), and bitwise
     equal to the resident kernel forced through renet_debug_gemm on the same operands.
  2. layer-1 gather: per row within (n + 4) 2^-24 sum |term| (rgcn_contract_check's bar, n = the row's in-degree); rows
     without in-edges keep ReLU(self-loop row) bit for bit.
  3. read-out sub-graph: uniq[:U] ascending and distinct, uniq[readout_c[i]] == readout[i], the copied norms equal the
     parent's; layer 2's self-loop and gather restated from the PARENT CSR (all in-edges of uniq[u], the parent's norm),
     per row as in 1-2; rows U..S follow the padding contract (uniq 0, norm 1, no edges: H2 = the self-loop row of node 0).
  4. renet_gru_fwd from the kernel's own H2: every row of hn4 and hn3 within tau = 1e-4 (encoder_contract_check.row_ratio).
  5. end to end: hn against a float64 chain from ent through all four stages (layer 1's ReLU taken at the kernel's H1 > 0).
  6. renet_rgcn_block_bwd on layer 1 (tile dH, d200 dW, split-K dW_loop), default and deterministic mode (two runs bitwise
     equal): dH and dW per row within the rgcn bar, dW_loop per row within 2e-5 (|ref row| + 1e-2 |ref|).
  7. renet_rgcn_bipartite_bwd on the read-out sub-graph, both modes, per row within the rgcn bar.
  6-7, dW: the rgcn bar grows with the relation's edge count n, and relation 0 has 2 M edges: there (n + 4) 2^-24 is 0.12,
     loose enough to miss half of the relation's 64-edge runs going missing (a random-sign sum of n terms is ~ sqrt(n) of
     a term, the bar ~ n).  Each dW row is therefore also held to TAU_DW = 1e-4 (|ref row| + 1e-2 |ref|), what fp32
     summation in runs of 64 edges gives (~ 1e-5 of the row at 31 k runs) with margin.
  8. renet_gru_bwd at Q = 32 768: dH2, d_ent, d_rel, d_glob and every GRU parameter gradient per row within tau = 5e-4.
Accumulated outputs start from a random non-zero base; written ones start as NaN.

Premises asserted on the host before any launch is checked: layer 1 is above kStreamMaxNodes, its largest in-degree and the
number of destinations heavier than one warp's share of their 16-row tile; relation 0 spans many 64-edge dW runs; U < S;
the recurrence walks >= 28 m-tiles per CTA.  Serving kernels are read from torch.profiler traces.

Discriminating power: before any GPU comparison, five plausible mistakes are applied to the float64 restatement and each
must miss its stage's bar by >= 10x on every targeted row (layer-1 mistakes on the first 2^16 destinations):
  no-node-ent  layer 1 reads source rows without node_ent (every row with in-edges)
  rev-type     one in-edge of each row of in-degree 1..32 takes its reverse-direction type (r +- R)
  norm-next    a read-out row takes the neighbouring node's norm (rows of in-degree 1..32 whose neighbour's norm differs;
               on a hub of thousands of edges next to a node of nearly the same degree the change is within rounding)
  glob-next    a sequence's last read-out row reads the next component's glob row (64 sequences)
  mtile-prev   the recurrence reads h_{t-1} of the neighbouring 128-row m-tile (the 128 rows of m-tile 1)

usage: synth_contract_check.py [--nodes N] [--forward-only].  Prints SYNTH_CONTRACT_OK on success."""
import argparse
import os
import re
import sys
import time
import traceback
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [ROOT, HERE]
import bench_synth  # noqa: E402
import encoder_contract_check as ec  # noqa: E402
import rgcn_contract_check as rc  # noqa: E402
from oracle import restate  # noqa: E402
from renet_b200 import _lib  # noqa: E402

DEV = rc.DEV
H, NB = bench_synth.H_DIM, bench_synth.NUM_BASES
G, R, Q, SL, SEED = 250, 500, 32768, 10, 999
R2 = 2 * R
CHUNK = 1 << 19            # edges per float64 pass
BLOCK = 1 << 19            # destinations per float64 restatement of layer 1
MROWS = 1 << 16            # destinations the layer mistakes are restated on
MISS = 10.0
TAU_LOOP = 2e-5            # dW_loop per row (rgcn_contract_check's dWloop bar, per row)
TAU_DW = 1e-4              # dW per relation row, relative to the row (module docstring)
RESIDENT, DEDUP = 5, 6
with open(os.path.join(ROOT, 'renet_b200', 'csrc', 'common.cuh')) as _fh:
    _src = _fh.read()
STREAM_MAX_NODES = int(re.search(r'kStreamMaxNodes = (\d+);', _src).group(1))
DEDUP_MIN_ROWS = int(re.search(r'kDedupMinRows = (\d+);', _src).group(1))

L, P = _lib.lib(), _lib.ptr
RATIOS = {}                # stage / gradient -> largest err / bar
MISSES = {}                # mistake -> smallest miss / bar over its targeted rows
SERVED = {}                # stage -> kernels that served it
FAILED = []


def stage(name):
    """run a check; a failure is recorded and the remaining checks still run (every number of one run is reported)"""
    def wrap(fn):
        t0 = time.perf_counter()
        try:
            fn()
            print('%-28s ok   (%.1f s)' % (name, time.perf_counter() - t0), flush=True)
        except AssertionError as e:
            FAILED.append('%s: %s' % (name, e))
            print('%-28s FAILED: %s' % (name, e), flush=True)
            traceback.print_exc()
        return fn
    return wrap


def note(key, ratio):
    RATIOS[key] = max(RATIOS.get(key, 0.0), float(ratio))


def kernel_names(fn):
    """the library's kernels fn launches, by demangled name in launch order (torch's own kernels left out); fn runs between
    two torch kernels, as rgcn_contract_check.kernels_of does, so records lost at a trace's edges are torch's"""
    prime = torch.zeros(1, device=DEV)
    names = []
    for _ in range(5):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            prime.add_(1)
            torch.cuda.synchronize()
            fn()
            torch.cuda.synchronize()
            prime.add_(1)
            torch.cuda.synchronize()
        evs = [ev for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and 'at::' not in ev.name]
        names = [re.search(r'(\w+_kernel)', ev.name).group(1) for ev in sorted(evs, key=lambda ev: ev.time_range.start)
                 if re.search(r'\w+_kernel', ev.name)]
        if names:
            break
    return names


def served(key, fn, expect_rgcn=None, contains=(), absent=()):
    """expect_rgcn: the exact {(rgcn kernel, template booleans)} of rgcn_contract_check.kernels_of; contains: kernel names
    that must appear in this order; absent: names that must not appear"""
    names = kernel_names(fn)
    SERVED[key] = names
    if expect_rgcn is not None:
        seen = set()
        for _ in range(5):         # the union over traces: a trace can lose a record, never add one
            seen |= rc.kernels_of(fn)
            if seen == expect_rgcn:
                break
        SERVED[key] = sorted(seen)
        assert seen == expect_rgcn, '%s: ran %s, expected %s' % (key, sorted(seen), sorted(expect_rgcn))
    it = iter(names)
    assert all(any(n == c for n in it) for c in contains), '%s: %s do not run in this order: %s' % (key, contains, names)
    assert not set(absent) & set(names), '%s: %s ran' % (key, sorted(set(absent) & set(names)))


# ---- the shard, as bench_synth.run_synth1m builds it ------------------------------------------------------------------------
def build(N):
    from renet_b200.graph import ReadoutSubgraph, build_csr
    from renet_b200.gru import _gru_params
    from renet_b200.model import RENet
    s = types.SimpleNamespace(N=N)
    dev = torch.device(DEV)
    sh = bench_synth.make_shard(torch, N, G, R, Q, SL, SEED, dev)
    s.sh, s.E = sh, int(sh['src'].numel())
    s.S = Q * SL
    s.row_ptr, s.col_src, s.col_type, _ = build_csr(sh['dst'], sh['src'], sh['type_s'], N)
    deg = (s.row_ptr[1:] - s.row_ptr[:-1]).float().clamp_(min=1)
    s.norm = 1.0 / deg

    class _G:      # the surface ReadoutSubgraph reads
        pass
    g = _G()
    g.device, g.N, g.row_ptr, g.col_src, g.norm = dev, N, s.row_ptr, s.col_src, s.norm
    g.col_type = lambda reverse: s.col_type
    g.hot_rel = lambda reverse: None
    s.sub = ReadoutSubgraph(g, sh['readout'], False)
    s.U, s.E2 = s.sub.sizes()
    torch.manual_seed(999)
    s.ent = torch.randn(N, H, device=dev) * 0.1
    s.node_ent = torch.randperm(N, device=dev).to(torch.int32)
    m = RENet(1024, H, R, dropout=0).to(dev).eval()
    s.W1, s.L1, s.W2, s.L2 = (m.aggregator.rgcn1.weight.detach(), m.aggregator.rgcn1.loop_weight.detach(),
                              m.aggregator.rgcn2.weight.detach(), m.aggregator.rgcn2.loop_weight.detach())
    s.rel = torch.randn(R, H, device=dev) * 0.1
    s.glob = torch.randn(G, H, device=dev) * 0.1
    s.seq_r = torch.randint(0, R, (Q,), device=dev, dtype=torch.int32)
    s.seq_len = torch.full((Q,), SL, dtype=torch.int32, device=dev)
    s.seq_start = (torch.arange(Q, device=dev) * SL).to(torch.int32)
    s.bs = np.full(SL, Q, dtype=np.int32)
    s.nbytes = int(L.renet_gru_workspace_bytes(s.S, Q, G, H))
    s.ws = torch.empty(s.nbytes // 4 + 4, dtype=torch.float32, device=dev)
    s.p4 = [t.detach() for t in _gru_params(m.encoder)]
    s.p3 = [t.detach() for t in _gru_params(m.encoder_r)]
    s.stream = _lib.stream()
    # the parent graph's edges in CSR order, and the read-out sub-graph restated from the parent CSR
    s.deg = (s.row_ptr[1:] - s.row_ptr[:-1]).long()
    s.dst = torch.repeat_interleave(torch.arange(N, device=dev), s.deg, output_size=s.E)
    s.g1 = types.SimpleNamespace(src=s.col_src, dst=s.dst, et=s.col_type, n_src=N, n_dst=N, E=s.E, R2=R2)
    flag = torch.zeros(N, dtype=torch.bool, device=dev)
    flag[sh['readout'].long()] = True
    s.uniq_p = flag.nonzero().flatten()
    pos = torch.cumsum(flag.long(), 0) - 1
    keep = flag[s.dst]
    s.uniq_pad = torch.zeros(s.S, dtype=torch.long, device=dev)
    s.uniq_pad[:len(s.uniq_p)] = s.uniq_p
    s.norm2 = torch.ones(s.S, device=dev)
    s.norm2[:len(s.uniq_p)] = s.norm[s.uniq_p]
    s.g2 = types.SimpleNamespace(src=s.col_src[keep], dst=pos[s.dst[keep]], et=s.col_type[keep], n_src=N, n_dst=s.S,
                                 E=int(keep.sum()), R2=R2)
    s.deg2 = torch.bincount(s.g2.dst, minlength=s.S)
    del flag, pos, keep
    return s


def premises(s):
    N = s.N
    assert N > STREAM_MAX_NODES, 'layer 1 would run on the stream gather'
    rp = s.row_ptr.long()
    tiles = (N + 15) // 16
    ends = torch.clamp(torch.arange(tiles + 1, device=DEV) * 16, max=N)
    te = rp[ends[1:]] - rp[ends[:-1]]
    share = (te + 7) // 8                                    # one warp's slice of its tile's edges (rgcn_tile.cuh)
    heavy = int((s.deg > share[torch.arange(N, device=DEV) // 16]).sum())
    max_deg = int(s.deg.max())
    rel0 = int((s.col_type == 0).sum())
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    mtiles = (Q + 127) // 128
    gz = max(1, min(mtiles, sms // (2 * ((H + 31) // 32))))
    print('shard: N = %d, E = %d, tile grid %d CTAs, max in-degree %d, %d destinations heavier than a warp\'s share of '
          'their tile, relation 0: %d edges (%d dW runs of 64), U = %d of S = %d, E2 = %d (E_cap %d), recurrence grid '
          '(7, 2, %d): %d m-tiles, %d-%d per CTA' % (N, s.E, tiles, max_deg, heavy, rel0, -(-rel0 // 64), s.U, s.S, s.E2,
                                                      s.sub.E_cap, gz, mtiles, mtiles // gz, -(-mtiles // gz)), flush=True)
    assert max_deg > 1000 and heavy >= G, (max_deg, heavy)       # at least each component's first row
    assert rel0 > 64 * 1000, rel0
    assert 0 < s.U < s.S and s.S >= DEDUP_MIN_ROWS and N >= DEDUP_MIN_ROWS
    assert mtiles // gz >= 28, (mtiles, gz)


# ---- the step's calls ---------------------------------------------------------------------------------------------------------
def selfloop(A, idx, B, M, s):
    out = torch.full((M, H), float('nan'), device=DEV)
    _lib.check(L.renet_selfloop_gemm(P(A), P(idx), P(B), P(out), M, H, H, s.stream), 'selfloop')
    return out


def debug_gemm(kernel, A, idx, B, M, s):
    out = torch.full((M, H), float('nan'), device=DEV)
    ws = torch.empty(-(-H // 200) * -(-H // 32) * 53248, dtype=torch.uint8, device=DEV)
    got = L.renet_debug_gemm(0, kernel, P(A), P(idx), H, P(B), H, P(out), H, None, M, H, H, 0, 1, 0, 0, 0, P(ws), ws.numel(),
                             s.stream)
    if got < 0:
        _lib.check(got, 'renet_debug_gemm')
    return got, out


def gather1(s, loop_rows):
    out = loop_rows.clone()
    _lib.check(L.renet_rgcn_gather(P(s.ent), P(s.node_ent), P(s.W1), P(s.row_ptr), P(s.col_src), P(s.col_type), P(s.norm),
                                   P(out), s.N, s.E, H, H, NB, R2, 1, 1, s.stream), 'gather1')
    return out


def gather2(s, H1, loop_rows):
    sub = s.sub
    out = loop_rows.clone()
    _lib.check(L.renet_rgcn_gather(P(H1), None, P(s.W2), P(sub.row_ptr), P(sub.col_src), P(sub.col_type(False)), P(sub.norm),
                                   P(out), s.S, sub.E_cap, H, H, NB, R2, 0, 1, s.stream), 'gather2')
    return out


def gru_fwd(s, H2):
    hn = torch.full((2, Q, H), float('nan'), device=DEV)
    p4, p3 = s.p4, s.p3
    rc_ = L.renet_gru_fwd(P(H2), P(s.sub.readout_c), P(s.sh['row_glob']), P(s.glob), P(s.ent), P(s.rel), P(s.sh['seq_s']),
                          P(s.seq_r), P(s.seq_len), P(s.seq_start), s.bs.ctypes.data_as(_lib.ctypes.c_void_p), SL, P(p4[0]),
                          P(p4[1]), P(p4[2]), P(p4[3]), P(p3[0]), P(p3[1]), P(p3[2]), P(p3[3]), P(hn[0]), P(hn[1]), s.S, Q, G,
                          H, P(s.ws), s.nbytes, s.stream)
    _lib.check(rc_, 'gru')
    return hn


# ---- float64 ------------------------------------------------------------------------------------------------------------------
def selfloop64(A, idx, B, a, b):
    rows = (A[idx[a:b].long()] if idx is not None else A[a:b]).double()
    return rows @ B.double(), rows.abs() @ B.double().abs()


def layer1_blocks(s, loop_rows):
    """layer 1 restated per block of BLOCK destinations: yields (a, b, pre-activation, S) of rows [a, b);
    loop_rows(a, b): the block's self-loop rows"""
    rp = s.row_ptr.long()
    for a in range(0, s.N, BLOCK):
        b = min(s.N, a + BLOCK)
        e0, e1 = int(rp[a]), int(rp[b])
        loop = loop_rows(a, b)
        g = types.SimpleNamespace(src=s.col_src[e0:e1], dst=s.dst[e0:e1] - a, et=s.col_type[e0:e1], n_src=s.N, n_dst=b - a,
                                  E=e1 - e0, R2=R2)
        if g.E == 0:                               # ref_forward's E = 0 case is the pass-through of a whole graph
            yield a, b, loop.double(), loop.double().abs()
        else:
            pre, S_ = rc.ref_forward(g, s.ent, s.node_ent, s.W1, s.norm[a:b], loop, CHUNK)
            yield a, b, pre, S_


def first_rows(g, rp, n):
    """the sub-graph of g's edges into destinations < n (g's edges are in destination order)"""
    e = int(rp[n])
    return types.SimpleNamespace(src=g.src[:e], dst=g.dst[:e], et=g.et[:e], n_src=g.n_src, n_dst=n, E=e, R2=g.R2)


def gru_inputs(s, H2, ent, rel, glob, row_glob=None):
    """restate.packed_inputs; ent: the whole table, of which only the Q sequences' rows are read (a float64 copy of the
    table would be 6.7 GB at 4 M nodes)"""
    rg = (s.sh['row_glob'] if row_glob is None else row_glob).long()
    lens = np.full(Q, SL, dtype=np.int64)
    ent_q = ent[s.sh['seq_s'].long()].double()
    X4, X3, _, _ = restate.packed_inputs(H2, s.sub.readout_c.long(), lens, torch.arange(Q, device=DEV), s.seq_r.long(), ent_q,
                                         rel, glob[rg])
    return X4, X3


def gru64(X, w_ih, w_hh, b_ih, b_hh, prev=None):
    """restate.gru_final_hidden_batched for Q sequences of length SL; prev: the row of h_{t-1} each sequence reads"""
    if prev is None:
        return restate.gru_final_hidden_batched(X, np.full(Q, SL, dtype=np.int64), w_ih, w_hh, b_ih, b_hh)
    gi = (X @ w_ih.t() + b_ih).view(Q, SL, -1)
    h = torch.zeros(Q, H, dtype=X.dtype, device=X.device)
    for t in range(SL):
        hp = h[prev]
        gh = hp @ w_hh.t() + b_hh
        r = torch.sigmoid(gi[:, t, :H] + gh[:, :H])
        z = torch.sigmoid(gi[:, t, H:2 * H] + gh[:, H:2 * H])
        n = torch.tanh(gi[:, t, 2 * H:] + r * gh[:, 2 * H:])
        h = (1 - z) * n + z * hp
    return h


def d64(ps):
    return [t.double() for t in ps]


def gru_miss(h4, h3, ref4, ref3, targets):
    r = torch.maximum(ec.row_ratio(h4, ref4, ec.TAU_FWD), ec.row_ratio(h3, ref3, ec.TAU_FWD))
    return float(r[targets].min())


def mistakes(s, H1_64, sl2_64, H2_64, ref4, ref3):
    relu = lambda t: t.clamp_min(0)
    rp = s.row_ptr.long()
    M = min(MROWS, s.N)
    g1m = first_rows(s.g1, rp, M)
    sl1_64 = selfloop64(s.ent, s.node_ent, s.L1, 0, M)[0]
    ref, S1 = rc.ref_forward(g1m, s.ent, s.node_ent, s.W1, s.norm[:M], sl1_64, CHUNK)
    n1 = s.deg[:M]
    has = (n1 > 0).nonzero().flatten()
    mut, _ = rc.ref_forward(g1m, s.ent, None, s.W1, s.norm[:M], sl1_64, CHUNK)
    MISSES['no-node-ent'] = float(rc.bar_ratio(relu(mut), relu(ref), S1, n1)[0][has].min())
    tgt = ((n1 >= 1) & (n1 <= 32)).nonzero().flatten()
    et = g1m.et.clone()
    first = rp[tgt]
    et[first] = (et[first] + R) % R2
    mut, _ = rc.ref_forward(types.SimpleNamespace(**{**vars(g1m), 'et': et}), s.ent, s.node_ent, s.W1, s.norm[:M],
                            sl1_64, CHUNK)
    MISSES['rev-type'] = float(rc.bar_ratio(relu(mut), relu(ref), S1, n1)[0][tgt].min())
    # layer 2: the neighbouring node's norm, on the first M2 compact rows
    M2 = min(MROWS, s.U)
    rp2 = torch.cat((torch.zeros(1, dtype=torch.long, device=DEV), torch.cumsum(s.deg2, 0)))
    g2m = first_rows(s.g2, rp2, M2)
    ref2, S2 = rc.ref_forward(g2m, H1_64, None, s.W2, s.norm2[:M2], sl2_64[:M2], CHUNK)
    nxt = torch.clamp(s.uniq_pad[:M2] + 1, max=s.N - 1)
    norm_m = s.norm[nxt]
    n2 = s.deg2[:M2]
    tgt = ((n2 >= 1) & (n2 <= 32) & (norm_m != s.norm2[:M2])).nonzero().flatten()
    mut, _ = rc.ref_forward(g2m, H1_64, None, s.W2, norm_m, sl2_64[:M2], CHUNK)
    MISSES['norm-next'] = float(rc.bar_ratio(mut, ref2, S2, s.deg2[:M2])[0][tgt].min())
    del ref, S1, mut, ref2, S2
    # GRU: the next component's glob row at the last step of 64 sequences; the neighbouring m-tile's h_{t-1}
    glob64, rel64 = s.glob.double(), s.rel.double()
    p4, p3 = d64(s.p4), d64(s.p3)
    seqs = torch.linspace(0, Q - 1, 64, device=DEV).round().long()
    rg = s.sh['row_glob'].clone()
    last = seqs * SL + SL - 1
    rg[last] = (rg[last] + 1) % G
    X4, X3 = gru_inputs(s, H2_64, s.ent, rel64, glob64, rg)
    MISSES['glob-next'] = gru_miss(gru64(X4, *p4), gru64(X3, *p3), ref4, ref3, seqs)
    X4, X3 = gru_inputs(s, H2_64, s.ent, rel64, glob64)
    prev = torch.arange(Q, device=DEV)
    prev[128:256] += 128
    MISSES['mtile-prev'] = gru_miss(gru64(X4, *p4, prev=prev), gru64(X3, *p3, prev=prev), ref4, ref3,
                                    torch.arange(128, 256, device=DEV))
    for k, v in sorted(MISSES.items()):
        print('mistake %-12s misses its bar by %.3g x (smallest over its targeted rows)' % (k, v), flush=True)
    bad = {k: v for k, v in MISSES.items() if v < MISS}
    assert not bad, 'mistakes within %g x of the bar: %s' % (MISS, bad)


# ---- the run ------------------------------------------------------------------------------------------------------------------
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--nodes', type=int, default=1000000)
    ap.add_argument('--forward-only', action='store_true')
    args = ap.parse_args()
    t_start = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    free0 = torch.cuda.mem_get_info()[0] / 2 ** 30
    s = build(args.nodes)
    N, S, U = s.N, s.S, s.U
    premises(s)
    relu = lambda t: t.clamp_min(0)

    # ---- the benchmarked step's five calls, in its order
    H1sl = selfloop(s.ent, s.node_ent, s.L1, N, s)
    H1 = gather1(s, H1sl)
    H2sl = selfloop(H1, s.sub.uniq, s.L2, S, s)
    H2 = gather2(s, H1, H2sl)
    hn = gru_fwd(s, H2)
    torch.cuda.synchronize()

    # ---- float64 chain from ent (layer 1's ReLU at the kernel's H1 > 0), then the mistakes, before any comparison
    with torch.no_grad():
        H1_64 = torch.empty(N, H, dtype=torch.float64, device=DEV)
        for a, b, pre, _ in layer1_blocks(s, lambda a, b: selfloop64(s.ent, s.node_ent, s.L1, a, b)[0]):
            H1_64[a:b] = pre * (H1[a:b] > 0)
        del pre
        sl2_64 = H1_64[s.uniq_pad] @ s.L2.double()
        H2_64, _ = rc.ref_forward(s.g2, H1_64, None, s.W2, s.norm2, sl2_64, CHUNK)
        X4, X3 = gru_inputs(s, H2_64, s.ent, s.rel.double(), s.glob.double())
        e2e4, e2e3 = gru64(X4, *d64(s.p4)), gru64(X3, *d64(s.p3))
        del X4, X3

        @stage('mistakes (fp64)')
        def _():
            mistakes(s, H1_64, sl2_64, H2_64, e2e4, e2e3)
        del H1_64, sl2_64, H2_64

        # ---- 1. layer-1 self-loop
        @stage('1 self-loop layer 1')
        def _():
            served('self-loop 1', lambda: selfloop(s.ent, s.node_ent, s.L1, N, s),
                   contains=('dedup_insert_kernel', 'umma_gemm_resident_kernel', 'dedup_expand_kernel'))
            check_selfloop('self-loop 1', H1sl, s.ent, s.node_ent, s.L1, N, s)

        # ---- 2. layer-1 gather
        @stage('2 gather layer 1')
        def _():
            served('gather 1', lambda: gather1(s, H1sl), rc.fwd_kernel('tile', True, True, True))
            rc.WORST.clear()
            for a, b, pre, S1 in layer1_blocks(s, lambda a, b: H1sl[a:b]):
                rc.check_rows('gather 1', 'synth rows %d..%d' % (a, b), 'gather 1', H1[a:b], relu(pre), S1, s.deg[a:b],
                              relu(H1sl[a:b]))
            note('gather 1', rc.WORST['gather 1'][0])

        # ---- 3. read-out sub-graph and layer 2
        @stage('3 read-out sub-graph')
        def _():
            sub = s.sub
            uniq = sub.uniq.long()
            assert U == len(s.uniq_p) and s.E2 == s.g2.E, ((U, len(s.uniq_p)), (s.E2, s.g2.E))
            assert bool((uniq[1:U] > uniq[:U - 1]).all()), 'uniq[:U] is not ascending and distinct'
            assert torch.equal(uniq[:U], s.uniq_p)
            rc_ = sub.readout_c.long()
            assert bool((rc_ < U).all()) and torch.equal(uniq[rc_], s.sh['readout'].long()), 'uniq[readout_c[i]] != readout[i]'
            assert torch.equal(sub.norm[:U], s.norm[uniq[:U]]), 'copied norms differ from the parent\'s'
            rp2 = sub.row_ptr.long()
            assert torch.equal(rp2[1:] - rp2[:-1], s.deg2), 'in-degrees differ from the parent CSR\'s'
            # padding: unused capacity is valid, edge-less rows of node 0 with norm 1
            assert bool((uniq[U:] == 0).all()) and bool((sub.norm[U:] == 1).all()) and bool((rp2[U:] == s.E2).all())

        @stage('3 self-loop layer 2')
        def _():
            served('self-loop 2', lambda: selfloop(H1, s.sub.uniq, s.L2, S, s),
                   contains=('dedup_insert_kernel', 'umma_gemm_resident_kernel', 'dedup_expand_kernel'))
            check_selfloop('self-loop 2', H2sl, H1, s.uniq_pad, s.L2, S, s, idx_kernel=s.sub.uniq)

        @stage('3 gather layer 2')
        def _():
            served('gather 2', lambda: gather2(s, H1, H2sl), rc.fwd_kernel('tile', False, True, False))
            ref, S2 = rc.ref_forward(s.g2, H1, None, s.W2, s.norm2, H2sl, CHUNK)
            check('gather 2', H2, ref, S2, s.deg2, H2sl)
            pad = H2[U:].contiguous().view(torch.int32)
            assert bool((pad == pad[:1]).all()) and torch.equal(H2[U:U + 1], H2sl[U:U + 1]), 'rows U..S are not node 0\'s row'

        # ---- 4. the fused read-out + GRU from the kernel's H2
        @stage('4 GRU forward')
        def _():
            served('GRU forward', lambda: gru_fwd(s, H2), contains=('gru_recur_kernel',), absent=('gru_gate_kernel',))
            X4, X3 = gru_inputs(s, H2.double(), s.ent, s.rel.double(), s.glob.double())
            check_gru('GRU forward', hn, gru64(X4, *d64(s.p4)), gru64(X3, *d64(s.p3)))

        # ---- 5. end to end
        @stage('5 end to end')
        def _():
            check_gru('end to end', hn, e2e4, e2e3)
        del e2e4, e2e3

    if not args.forward_only:
        backward(s, H1, H2, hn)

    wall = time.perf_counter() - t_start
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print('\nsynth shard N = %d on %s: %s' % (N, torch.cuda.get_device_name(0), 'forward only' if args.forward_only else
                                              'forward and backward'))
    for k, v in RATIOS.items():
        print('  %-34s worst err / bar %.3f' % (k, v))
    for k, v in SERVED.items():
        print('  served %-20s %s' % (k, v))
    print('  wall time %.1f s, peak memory %.1f GB (torch.cuda.max_memory_allocated; %.1f GB free at the start)' % (
        wall, peak, free0), flush=True)
    assert not FAILED, 'failed:\n  ' + '\n  '.join(FAILED)
    print('SYNTH_CONTRACT_OK N = %d' % N)


def check(key, got, ref, S, n, exact_to):
    """rgcn_contract_check.check_rows over chunks of rows (its temporaries are three float64 copies of the rows)"""
    rc.WORST.clear()
    step = 1 << 19
    for a in range(0, len(got), step):
        b = min(len(got), a + step)
        rc.check_rows(key, 'synth rows %d..%d' % (a, b), key, got[a:b], ref[a:b], S[a:b], n[a:b], exact_to[a:b])
    note(key, rc.WORST[key][0])


def check_selfloop(key, got, A, idx, B, M, s, idx_kernel=None):
    """per row against fp64 (idx: the restatement's rows), and bitwise equal to the resident kernel on the kernel's own
    operands (idx_kernel, default idx)"""
    idx_kernel = idx if idx_kernel is None else idx_kernel
    assert not torch.isnan(got).any(), key + ': rows left unwritten'
    worst = 0.0
    step = 1 << 18
    for a in range(0, M, step):
        b = min(M, a + step)
        ref, S_ = selfloop64(A, idx, B, a, b)
        r, _ = rc.bar_ratio(got[a:b], ref, S_, torch.full((b - a,), H, dtype=torch.long, device=DEV))
        worst = max(worst, float(r.max()))
    note(key, worst)
    assert worst <= rc.C, '%s: %.3g x (K + 4) 2^-24 sum |a b| off' % (key, worst)
    k0, via = debug_gemm(0, A, idx_kernel, B, M, s)
    assert k0 == DEDUP and torch.equal(via.view(torch.int32), got.view(torch.int32)), (key, 'dispatch', k0)
    k, res = debug_gemm(RESIDENT, A, idx_kernel, B, M, s)
    assert k == RESIDENT, (key, k)
    assert torch.equal(res.view(torch.int32), got.view(torch.int32)), '%s: not bitwise equal to the resident kernel' % key


def check_gru(key, hn, ref4, ref3):
    assert not torch.isnan(hn).any(), key + ': hidden states left unwritten'
    for what, got, ref in (('hn4', hn[0], ref4), ('hn3', hn[1], ref3)):
        r = ec.row_ratio(got, ref, ec.TAU_FWD)
        worst = float(r.max())
        note('%s %s' % (key, what), worst)
        assert worst <= 1.0, '%s %s: row %d is %.3g x the bar off; %d rows fail' % (key, what, int(r.argmax()), worst,
                                                                                   int((r > 1).sum()))


def check_grad(key, got, base, ref, tau=ec.TAU_GRAD):
    """an accumulated gradient (base None: written) per row: rows exactly 0 in fp64 must come back as the base bit for bit"""
    g = got.double() - (base.double() if base is not None else 0)
    g, r = (g.reshape(1, -1), ref.reshape(1, -1)) if ref.dim() == 1 else (g, ref)
    zero = (r == 0).all(1)
    if base is not None:
        b = base.reshape(g.shape)
        untouched = (got.reshape(g.shape) != b).any(1) & zero
        assert not bool(untouched.any()), '%s: row %d is 0 in fp64 but not the base' % (key, int(untouched.nonzero()[0]))
    ratio = ec.row_ratio(g, r, tau)
    worst = float(ratio.max())
    note(key, worst)
    assert worst <= 1.0, '%s: row %d is %.3g x the bar off; %d of %d rows fail' % (key, int(ratio.argmax()), worst,
                                                                                  int((ratio > 1).sum()), len(ratio))


# ---- backward -----------------------------------------------------------------------------------------------------------------
def backward(s, H1, H2, hn):
    from renet_b200.graph import build_csr
    N, S = s.N, s.S
    gen = torch.Generator(device=DEV).manual_seed(SEED + 1)

    # ---- 6. layer 1: renet_rgcn_block_bwd (tile dH, d200 dW, split-K dW_loop)
    dst32 = s.dst.to(torch.int32)
    t1 = build_csr(s.col_src, dst32, s.col_type, N)[:3]
    r1 = build_csr(s.col_type, s.col_src, dst32, R2)[:3]
    del dst32
    dout = torch.randn(N, H, device=DEV, generator=gen)
    base_W = torch.randn(R2, 400, device=DEV, generator=gen) * 1e-2
    base_Wl = torch.randn(H, H, device=DEV, generator=gen) * 1e-2
    ws = torch.empty(N * H + H * H, device=DEV)

    def call1():
        dH = torch.full((N, H), float('nan'), device=DEV)
        dW, dWl = base_W.clone(), base_Wl.clone()
        _lib.check(L.renet_rgcn_block_bwd(P(s.ent), P(s.node_ent), P(s.W1), P(s.L1), *[P(t) for t in t1], *[P(t) for t in r1],
                                          P(s.norm), P(H1), P(dout), P(dH), P(dW), P(dWl), P(ws), N, s.E, H, H, NB, R2, 1,
                                          s.stream), 'block bwd')
        return dH, dW, dWl

    Pm = dout * (H1 > 0)
    dH_loop = torch.zeros(N, H, device=DEV)
    _lib.check(L.renet_selfloop_gemm_bwd(P(s.ent), P(s.node_ent), P(s.L1), P(Pm), P(dH_loop), P(torch.zeros(H, H, device=DEV)),
                                         P(torch.empty(H * H, device=DEV)), N, H, H, s.stream), 'selfloop bwd')
    with torch.no_grad():
        rH, sH, rW, sW = rc.ref_backward(s.g1, s.ent, s.node_ent, s.W1, s.norm, Pm, CHUNK // 2)
        rH += dH_loop.double()
        sH += dH_loop.double().abs()
        Xr = s.ent[s.node_ent.long()].double()
        refl = Xr.t() @ Pm.double()
        del Xr
    out_deg = torch.bincount(s.col_src.long(), minlength=N)
    rel_n = torch.bincount(s.col_type.long(), minlength=R2)
    for det in (False, True):
        tag = ' det' if det else ''

        @stage('6 layer-1 backward' + tag)
        def _():
            with rc.deterministic(det):
                dH, dW, dWl = call1()
                if det:
                    again = call1()
                    assert all(torch.equal(a, b) for a, b in zip((dH, dW, dWl), again)), 'deterministic mode: two runs differ'
                    del again
                served('layer-1 bwd' + tag, call1, rc.bwd_kernels('tile', True, True, det))
            check('layer-1 dH' + tag, dH, rH, sH, out_deg, dH_loop)
            check('layer-1 dW' + tag, dW, rW + base_W.double(), sW + base_W.double().abs(), rel_n, base_W)
            check_grad('layer-1 dW row-relative' + tag, dW, base_W, rW, TAU_DW)
            check_grad('layer-1 dW_loop' + tag, dWl, base_Wl, refl, TAU_LOOP)
    del rH, sH, rW, sW, refl, Pm, dH_loop, ws, t1, r1, dout

    # ---- 7. layer 2: renet_rgcn_bipartite_bwd on the read-out sub-graph
    structs = s.sub.backward_structs(False, R2)
    dout2 = torch.randn(S, H, device=DEV, generator=gen)
    base_W2 = torch.randn(R2, 400, device=DEV, generator=gen) * 1e-2
    ws2 = torch.empty(S * H, device=DEV)

    def call2():
        dH = torch.full((N, H), float('nan'), device=DEV)
        dW = base_W2.clone()
        _lib.check(L.renet_rgcn_bipartite_bwd(P(H1), P(s.W2), *[P(t) for t in structs], P(s.sub.norm), P(H2), P(dout2), P(dH),
                                              P(dW), P(ws2), N, S, s.E2, H, H, NB, R2, 0, s.stream), 'bipartite bwd')
        return dH, dW

    with torch.no_grad():
        rH, sH, rW, sW = rc.ref_backward(s.g2, H1, None, s.W2, s.norm2, dout2, CHUNK // 2)
    out2 = torch.bincount(s.g2.src.long(), minlength=N)
    rel2 = torch.bincount(s.g2.et.long(), minlength=R2)
    for det in (False, True):
        tag = ' det' if det else ''

        @stage('7 layer-2 backward' + tag)
        def _():
            with rc.deterministic(det):
                dH, dW = call2()
                if det:
                    again = call2()
                    assert torch.equal(dH, again[0]) and torch.equal(dW, again[1]), 'deterministic mode: two runs differ'
                served('layer-2 bwd' + tag, call2, rc.bwd_kernels('tile', False, False, det))
            check('layer-2 dH' + tag, dH, rH, sH, out2, torch.zeros(N, H, device=DEV))
            check('layer-2 dW' + tag, dW, rW + base_W2.double(), sW + base_W2.double().abs(), rel2, base_W2)
            check_grad('layer-2 dW row-relative' + tag, dW, base_W2, rW, TAU_DW)
    del rH, sH, rW, sW, ws2, dout2

    # ---- 8. renet_gru_bwd at Q = 32 768 (the forward workspace holds renet_gru_fwd's state for H2)
    @stage('8 GRU backward')
    def _():
        gru_fwd(s, H2)
        dhn4 = torch.randn(Q, H, device=DEV, generator=gen)
        dhn3 = torch.randn(Q, H, device=DEV, generator=gen)
        leaves = {'H2': H2, 'ent': s.ent, 'rel': s.rel, 'glob': s.glob}
        names4 = ('w_ih4', 'w_hh4', 'b_ih4', 'b_hh4')
        names3 = ('w_ih3', 'w_hh3', 'b_ih3', 'b_hh3')
        leaves.update(zip(names4, s.p4))
        leaves.update(zip(names3, s.p3))
        lv = {k: v.double().requires_grad_(True) for k, v in leaves.items()}
        X4, X3 = gru_inputs(s, lv['H2'], lv['ent'], lv['rel'], lv['glob'])
        h4 = gru64(X4, *[lv[k] for k in names4])
        h3 = gru64(X3, *[lv[k] for k in names3])
        ((h4 * dhn4.double()).sum() + (h3 * dhn3.double()).sum()).backward()
        del X4, X3, h4, h3
        acc = {k: torch.randn(v.shape, device=DEV, generator=gen) * 1e-2 for k, v in leaves.items() if k != 'H2'}
        base = {k: v.clone() for k, v in acc.items()}
        dH2 = torch.full((S, H), float('nan'), device=DEV)
        bbytes = int(L.renet_gru_bwd_workspace_bytes(S, Q, G, H))
        bws = torch.empty(bbytes // 4 + 4, device=DEV)
        p4, p3 = s.p4, s.p3
        n0 = _lib.launch_count()

        def call():
            _lib.check(L.renet_gru_bwd(P(H2), P(s.sub.readout_c), P(s.sh['row_glob']), P(s.glob), P(s.ent), P(s.rel),
                                       P(s.sh['seq_s']), P(s.seq_r), P(s.seq_len), P(s.seq_start),
                                       s.bs.ctypes.data_as(_lib.ctypes.c_void_p), SL, P(p4[0]), P(p4[1]), P(p3[0]), P(p3[1]),
                                       P(dhn4), P(dhn3), P(dH2), P(acc['ent']), P(acc['rel']), P(acc['glob']),
                                       *[P(acc[k]) for k in names4 + names3], S, S, Q, G, H, P(s.ws), P(bws), bbytes,
                                       s.stream), 'gru bwd')
        call()
        torch.cuda.synchronize()
        SERVED['GRU backward'] = '%d launches' % (_lib.launch_count() - n0)
        check_grad('GRU dH2', dH2, None, lv['H2'].grad)
        for k in ('ent', 'rel', 'glob') + names4 + names3:
            check_grad('GRU d' + k, acc[k], base[k], lv[k].grad)


if __name__ == '__main__':
    main()
