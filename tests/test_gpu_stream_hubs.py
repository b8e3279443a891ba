"""-m gpu: hub source rows in the forward stream gather (renet_gather_stream_kernel with StCfg HUB > 0).

Layer 1 (input rows through an index) keeps each CTA's most frequent source nodes resident in shared memory: the
HUB = 64 most frequent of the kStHubBins = 2048 nodes from the CTA's smallest source, with at least 2 edges, ties at the
threshold to the smaller node ids.  Only where a source row is read from changes, so every case checks
  * on the host, that the graph has the property the case is about (a restatement of the kernel's CTA partition and
    hub choice);
  * from the profiled kernel names, that the stream kernel served it, with hub rows (layer 1) or without (plain input);
  * the float64 bar of rgcn_contract_check.run_fwd (and the caller's hot list giving the same result);
  * torch.equal against the same launch with the hub rows off (RENET_STREAM_CFG=3: 82 relation rows, no hubs).
"""
import os
import re

import numpy as np
import pytest
import torch

from rgcn_contract_check import DEV, Graph, ctas, mid_degrees, run_fwd
from test_stream_partition import warp_ranges

pytestmark = pytest.mark.gpu
HUB, BINS = 64, 2048
N = 20000                       # destinations: the stream kernel's size range for indexed input


def hub_choice(srcs):
    """the kernel's hub choice for one CTA's source nodes: {node}"""
    srcs = np.asarray(srcs, dtype=np.int64)
    if len(srcs) == 0:
        return set()
    lo = int(srcs.min())
    cnt = np.bincount(srcs[srcs < lo + BINS] - lo, minlength=BINS)
    c = np.minimum(cnt, 255)
    thr = next(t for t in range(2, 257) if (c >= t).sum() <= HUB)
    chosen = list(np.flatnonzero(c >= thr))
    if thr - 1 >= 2:
        chosen += list(np.flatnonzero(c == thr - 1)[:HUB - len(chosen)])
    return {lo + int(b) for b in chosen}


def cta_hubs(g):
    """[(cb, ce, hubs)] of the 132 CTAs"""
    return [(cb, ce, hub_choice(g.src[cb:ce])) for a, an, cb, ce in ctas(g.rp_dst)]


def stream_cfgs(fn):
    """the StCfg template arguments of the stream-kernel launches fn makes"""
    for _ in range(5):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            torch.zeros(1, device=DEV).add_(1)
            fn()
            torch.cuda.synchronize()
        names = [ev.name for ev in prof.events() if 'rgcn_gather_stream_kernel' in ev.name]
        if names:
            break
    cfgs = set()
    for nm in names:
        args = re.search(r'StCfg<([^>]*)>', nm).group(1).replace('(bool)', '').replace('false', '0').replace('true', '1')
        cfgs.add(tuple(int(x) for x in re.findall(r'\d+', args)))
    return cfgs


def launch(g, indexed, hot=None):
    from renet_b200 import _lib
    from rgcn_contract_check import fwd_structs, make_inputs
    L, P = _lib.lib(), _lib.ptr
    _, X, h_index, W, norm = make_inputs(g, indexed, 3)
    rp, cs, ct = fwd_structs(g)
    out = torch.zeros(g.n_dst, 200, device=DEV)
    if hot is None:
        rc = L.renet_rgcn_gather(P(X), P(h_index), P(W), P(rp), P(cs), P(ct), P(norm), P(out), g.n_dst, g.E, 200, 200, 100,
                                 g.R2, 1, 1, _lib.stream())
    else:
        rc = L.renet_rgcn_gather_hot(P(X), P(h_index), P(W), P(rp), P(cs), P(ct), P(norm), P(out), g.n_dst, g.E, 200, 200,
                                     100, g.R2, 1, 1, P(hot), hot.numel(), _lib.stream())
    _lib.check(rc, 'gather')


def check(case, g, indexed=True, hot_lists=((),)):
    """fp64 bar + hubs on == hubs off (torch.equal), each with and without the hot lists given"""
    from rgcn_contract_check import i32
    hub_cfg = (32, 2, 49, 0, 64) if indexed else (32, 2, 82, 0, 0)
    hots = [h for h in hot_lists if len(h)]
    for hot in [None] + [i32(h) for h in hots]:
        assert stream_cfgs(lambda: launch(g, indexed, hot)) == {hub_cfg}, case
    got = run_fwd(case, g, 'stream', True, True, indexed, hots=tuple(hots))
    os.environ['RENET_STREAM_CFG'] = '3'
    try:
        assert stream_cfgs(lambda: launch(g, indexed)) == {(32, 2, 82, 0, 0)}, case
        off = run_fwd(case + ' (no hubs)', g, 'stream', True, True, indexed, hots=tuple(hots))
    finally:
        del os.environ['RENET_STREAM_CFG']
    assert torch.equal(got, off), case


def by_sources(src, deg=None, R2=460, seed=0, n_src=N):
    deg = mid_degrees(N) if deg is None else deg
    dst = np.repeat(np.arange(len(deg)), deg)
    et = np.random.default_rng(seed).integers(0, R2, len(dst))
    return Graph(n_src, len(deg), R2, np.asarray(src(len(dst), dst)), dst, et)


def test_every_edge_from_one_source():
    g = by_sources(lambda E, dst: np.full(E, 7))
    assert all(h == {7} for cb, ce, h in cta_hubs(g) if ce > cb)
    check('one source', g)


def test_fewer_distinct_sources_than_hub():
    rng = np.random.default_rng(1)
    g = by_sources(lambda E, dst: rng.integers(100, 140, E))
    per = [len(np.unique(g.src[cb:ce])) for cb, ce, h in cta_hubs(g) if ce > cb]
    assert max(per) < HUB and min(per) > 1
    check('fewer sources than HUB', g)


def test_sources_outside_the_window():
    # near sources 0..299, and every fifth edge from 20 far nodes that are each the most frequent source of their CTA
    rng = np.random.default_rng(2)
    g = by_sources(lambda E, dst: np.where(np.arange(E) % 5 == 0, 10000 + rng.integers(0, 20, E), rng.integers(0, 300, E)))
    for cb, ce, h in cta_hubs(g):
        s = g.src[cb:ce]
        far = s[s >= s.min() + BINS]
        assert len(far) and np.bincount(far).max() > np.bincount(s[s < 300]).max() and not (h & set(far.tolist()))
    check('outside the window', g)


def test_hub_destination_cut_by_a_warp_boundary():
    deg = mid_degrees(N).copy()
    deg[5000] = 900                       # spans several warps of its CTA; all its edges come from node 3
    rng = np.random.default_rng(3)
    g = by_sources(lambda E, dst: np.where(dst == 5000, 3, rng.integers(0, N, E)), deg)
    rp = g.rp_dst
    a, an, cb, ce = next(c for c in ctas(rp) if c[0] <= 5000 < c[1])
    e0 = warp_ranges(rp, a, an, cb, ce)
    cut = [w for w in range(32) if e0[w] < e0[w + 1] and rp[5000] < e0[w] < rp[5001]]
    assert len(cut) >= 2 and 3 in hub_choice(g.src[cb:ce])
    check('hub cut by warps', g)


def test_resident_runs_across_index_blocks_and_all_or_no_resident_warps():
    # destinations in runs of ~300 edges from 8 hub nodes alternate with runs from sources used once
    deg = mid_degrees(N)
    rng = np.random.default_rng(4)

    def src(E, dst):
        run = (np.arange(E) // 300) % 2 == 0
        return np.where(run, rng.integers(50, 58, E), 1000 + np.arange(E) % (N - 1000))
    g = by_sources(src, deg, n_src=N)
    rp = g.rp_dst
    all_res = no_res = 0
    for (a, an, cb, ce), (_, _, hubs) in zip(ctas(rp), cta_hubs(g)):
        e0 = warp_ranges(rp, a, an, cb, ce)
        for w in range(32):
            res = np.isin(g.src[e0[w]:e0[w + 1]], list(hubs))
            if len(res) >= 16:
                all_res += bool(res.all())
                no_res += bool(not res.any())
    run = np.isin(g.src, np.arange(50, 58))
    longest = max(len(r) for r in np.split(run, np.flatnonzero(np.diff(run)) + 1) if r[0])
    assert all_res > 0 and no_res > 0 and longest >= 96
    check('runs across blocks', g)


def test_count_ties_at_the_hub_th_place():
    # every CTA: 100 sources of exactly 3 edges each among sources used once; 64 of the 100 are chosen, by node id
    deg = mid_degrees(N)
    E = int(deg.sum())
    src = 5000 + np.arange(E)                        # used once
    rng = np.random.default_rng(5)
    g0 = by_sources(lambda E_, dst: src, deg, n_src=5000 + E)
    for a, an, cb, ce in ctas(g0.rp_dst):
        pos = rng.choice(np.arange(cb, ce), min(300, ce - cb), replace=False)
        src[pos] = 1000 + (np.arange(len(pos)) // 3) + 100 * (a % 20)
    g = by_sources(lambda E_, dst: src, deg, n_src=5000 + E)
    tied = 0
    for cb, ce, h in cta_hubs(g):
        c = np.bincount(g.src[cb:ce] - g.src[cb:ce].min())
        if (c == 3).sum() > HUB and len(h) == HUB:
            tied += 1
    assert tied > 100
    check('ties', g)


@pytest.mark.parametrize('indexed', [True, False])
def test_benchmark_batch_with_and_without_the_hot_list(indexed):
    """bench.py's ICEWS18-shaped batch 0, subject side: layer 1's graph (indexed) and its structure with plain input rows"""
    from renet_b200 import hoststore, synthetic, utils
    tkg = synthetic.SyntheticTKG('icews18', seed=999, num_timestamps=240)
    gs = hoststore.GraphStore(tkg.graph_dict)
    q, sh, oh = tkg.batch(0, 1024, tail_only=False)
    hb = utils.assemble_history_batch(sh[0], sh[1], q[:, 0], tkg.graph_dict, torch.device(DEV))
    bg = hb.graph
    rp = bg.row_ptr.cpu().numpy().astype(np.int64)
    E = int(rp[-1])
    src, et = bg.col_src[:E].cpu().numpy(), bg.col_type(False)[:E].cpu().numpy()
    g = Graph(bg.N, bg.N, 2 * tkg.num_r, src, np.repeat(np.arange(bg.N), np.diff(rp)), et)
    assert 16384 <= g.n_dst <= 40960
    share = np.median([np.isin(g.src[cb:ce], list(h)).mean() for cb, ce, h in cta_hubs(g) if ce > cb])
    assert share > 0.3, share
    hot = gs.hot_relations(torch.device(DEV))[0].cpu().numpy()
    check('benchmark batch', g, indexed, hot_lists=((), hot))
