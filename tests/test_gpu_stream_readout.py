"""-m gpu: layer 2 on the read-out sub-graph (renet_readout_subgraph) through the kernel its size selects.

Read-out sub-graphs of benchmark-shaped batches (S ~ 8 k compact destinations, launched with the parent graph's edge
capacity) are served by the persistent stream gather.  On those, on a constructed one with a 150-edge hub and on one
without edges, the selected kernel is checked against
  * the tile kernel, which served these graphs before: max |diff| <= 1e-5 max |out| (the kernels sum a destination's
    edges in different associations);
  * a float64 restatement of the layer: max |diff| <= 2e-5 max |ref|;
and rows past S are left untouched.  Which kernel ran is read from the stream kernel's debug time stamps (written by the
stream kernel only).  The tile kernel is reached by launching with an edge count below the batch-scale threshold: it
reads the edges from row_ptr and uses the count for nothing else."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
EXTRA = 64                 # rows past S in the output buffer: must come back bit for bit


@pytest.fixture(scope='module')
def lib():
    from renet_b200 import _lib
    assert torch.cuda.is_available()
    return _lib


def _gather(_lib, H1, W, sub, reverse, loop, n_e, hot=None):
    """(out [S + EXTRA, 200], whether the stream kernel ran): layer 2 (linear, self-loop rows in the output) on sub"""
    L, P = _lib.lib(), _lib.ptr
    S = sub.N
    out = torch.full((S + EXTRA, 200), float('nan'), device=DEV)
    out[S:] = torch.arange(EXTRA * 200, device=DEV, dtype=torch.float32).view(EXTRA, 200) * 0.5 - 7.0
    out[:S] = loop
    stamps = torch.zeros(132 * 32 * 8, dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    L.renet_debug_stream_timing(P(stamps))
    try:
        if hot is None:
            rc = L.renet_rgcn_gather(P(H1), None, P(W), P(sub.row_ptr), P(sub.col_src), P(sub.col_type(reverse)), P(sub.norm),
                                     P(out), S, n_e, 200, 200, 100, W.shape[0], 0, 1, _lib.stream())
        else:
            rc = L.renet_rgcn_gather_hot(P(H1), None, P(W), P(sub.row_ptr), P(sub.col_src), P(sub.col_type(reverse)),
                                         P(sub.norm), P(out), S, n_e, 200, 200, 100, W.shape[0], 0, 1, P(hot), hot.numel(),
                                         _lib.stream())
        _lib.check(rc, 'gather')
        torch.cuda.synchronize()
    finally:
        L.renet_debug_stream_timing(None)
    return out, bool(stamps.any())


def _restate(H1, W, sub, reverse, loop):
    """float64: out[u] = norm[u] * sum_e blockdiag(W[type_e]) . H1[src_e] + loop[u]; rows without edges keep loop[u]"""
    U, E2 = sub.sizes()
    rp = sub.row_ptr.long()
    src, typ = sub.col_src[:E2].long(), sub.col_type(reverse)[:E2].long()
    dst = torch.repeat_interleave(torch.arange(sub.N, device=DEV), rp[1:] - rp[:-1])
    acc = torch.zeros(sub.N, 100, 2, dtype=torch.float64, device=DEV)
    for a in range(0, E2, 16384):                  # block b / in i / out j at b*4 + i*2 + j (RGCN.py:75-77)
        b = slice(a, min(a + 16384, E2))
        msg = torch.einsum('ebi,ebij->ebj', H1[src[b]].double().view(-1, 100, 2), W[typ[b]].double().view(-1, 100, 2, 2))
        acc.index_add_(0, dst[b], msg)
    return acc.view(sub.N, 200) * sub.norm.double()[:, None] + loop.double()


def _check(lib, H1, W, sub, reverse, hot, expect_stream):
    S = sub.N
    U, E2 = sub.sizes()
    gen = torch.Generator(device=DEV).manual_seed(S + E2)
    loop = torch.randn(S, 200, device=DEV, generator=gen) * 0.3          # stands in for the self-loop product
    got, ran_stream = _gather(lib, H1, W, sub, reverse, loop, sub.E_cap, hot)
    assert ran_stream == expect_stream, (S, sub.E_cap, ran_stream)
    tile, tile_stream = _gather(lib, H1, W, sub, reverse, loop, 1, hot)
    assert not tile_stream
    tail = torch.arange(EXTRA * 200, device=DEV, dtype=torch.float32).view(EXTRA, 200) * 0.5 - 7.0
    assert torch.equal(got[S:], tail) and torch.equal(tile[S:], tail)
    got, tile = got[:S], tile[:S]
    assert torch.isfinite(got).all()
    ref = _restate(H1, W, sub, reverse, loop)
    assert (got.double() - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    assert (got - tile).abs().max().item() <= 1e-5 * tile.abs().max().item()
    # destinations without edges (the padding between U and S among them) keep their self-loop row
    rp = sub.row_ptr.long()
    empty = (rp[1:] == rp[:-1]).nonzero().flatten()
    assert torch.equal(got[empty], loop[empty])
    return U, E2


def test_benchmark_shaped_readout_subgraphs(lib):
    """bench.py's ICEWS18-shaped batches 0 and 1, both directions; batch 0 with the dataset's relation ranking"""
    from renet_b200 import hoststore, synthetic, utils
    tkg = synthetic.SyntheticTKG('icews18', seed=999, num_timestamps=240)
    gs = hoststore.GraphStore(tkg.graph_dict)
    R2 = 2 * tkg.num_r
    torch.manual_seed(5)
    W = torch.randn(R2, 400, device=DEV) * 0.1
    max_deg = 0
    for i in (0, 1):
        q, sh, oh = tkg.batch(i, 1024, tail_only=False)
        for hist, col, reverse in ((sh, 0, False), (oh, 2, True)):
            hb = utils.assemble_history_batch(hist[0], hist[1], q[:, col], tkg.graph_dict, torch.device(DEV))
            g = hb.graph
            H1 = torch.randn(g.N, 200, device=DEV)
            sub = g.readout_sub(hb.readout, reverse)
            hot = gs.hot_relations(torch.device(DEV))[reverse] if i == 0 else None
            U, E2 = _check(lib, H1, W, sub, reverse, hot, expect_stream=True)
            assert 6000 < U <= sub.N and 50_000 < E2 < sub.E_cap
            rp = sub.row_ptr.cpu().numpy()
            max_deg = max(max_deg, int(np.diff(rp).max()))
    assert max_deg > 100          # the hubs of the read-out sub-graph are cut across warps


def _custom_subgraph(N, deg, readout, seed):
    """a batched graph with the given in-degrees (sources and relations random) and its read-out sub-graph"""
    from renet_b200.graph import ReadoutSubgraph

    class Graph:
        pass
    rng = np.random.default_rng(seed)
    g = Graph()
    g.device, g.N = torch.device(DEV), N
    rp = np.concatenate(([0], np.cumsum(deg))).astype(np.int32)
    E = int(rp[-1])
    g.row_ptr = torch.from_numpy(rp).to(DEV)
    g.col_src = torch.from_numpy(rng.integers(0, N, max(E, 1)).astype(np.int32)).to(DEV)
    ct = torch.from_numpy(rng.integers(0, 460, max(E, 1)).astype(np.int32)).to(DEV)
    g.col_type = lambda reverse: ct
    g.norm = torch.from_numpy((1.0 / np.maximum(deg, 1)).astype(np.float32)).to(DEV)
    return g, ReadoutSubgraph(g, torch.from_numpy(np.asarray(readout, dtype=np.int32)).to(DEV), False)


def test_constructed_hub_and_edgeless_readout_subgraphs(lib):
    N = 30000
    rng = np.random.default_rng(11)
    deg = rng.integers(0, 12, N)
    deg[[5, 20000]] = [150, 0]
    deg[25000:] = 0                                   # nodes without in-edges
    torch.manual_seed(7)
    W = torch.randn(460, 400, device=DEV) * 0.1
    H1 = torch.randn(N, 200, device=DEV)
    # 6 000 read-out rows (some repeated) over 5 000 distinct nodes, the 150-edge hub among them
    nodes = np.sort(np.concatenate(([5], rng.choice(np.arange(6, 25000), 4999, replace=False))))
    g, sub = _custom_subgraph(N, deg, np.concatenate((nodes, rng.choice(nodes, 1000))), 1)
    U, E2 = _check(lib, H1, W, sub, False, None, expect_stream=True)
    assert U == 5000 and E2 == deg[nodes].sum() and sub.N == 6000
    # every read-out node without in-edges: E2 = 0, all rows keep their self-loop rows
    g, sub = _custom_subgraph(N, deg, np.arange(25000, 29000), 2)
    assert sub.sizes() == (4000, 0)
    _check(lib, H1, W, sub, False, None, expect_stream=True)


def test_small_readout_subgraph_stays_on_the_tile_kernel(lib):
    N = 30000
    rng = np.random.default_rng(12)
    deg = rng.integers(0, 12, N)
    torch.manual_seed(8)
    W = torch.randn(460, 400, device=DEV) * 0.1
    H1 = torch.randn(N, 200, device=DEV)
    g, sub = _custom_subgraph(N, deg, rng.choice(N, 500, replace=False), 3)
    _check(lib, H1, W, sub, False, None, expect_stream=False)
