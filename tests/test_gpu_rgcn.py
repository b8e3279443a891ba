"""-m gpu: the CUDA RGCN block layer (through the C-ABI) against the reference's golden vectors and the
CPU oracle.  Tolerance: 1e-4 relative (max-abs-diff / max-abs-ref), the north-star bar; integer-valued
known-answer cases must be exact."""
import numpy as np
import pytest
import torch

from helpers import layer_case, load_npz, rel_err, t
from oracle import restate

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(scope='module')
def G():
    import gpu_helpers
    assert torch.cuda.is_available()
    return gpu_helpers


def _case_tensors(G, c):
    et = c['type_o'] if int(c['reverse']) else c['type_s']
    H, W = G.d(c['H']), G.d(c['W'])
    Wl = G.d(c['Wloop']) if bool(c['self_loop']) else None
    return H, W, Wl, et


def test_golden_layer_cases_forward(G):
    blob = load_npz('layer_cases.npz')
    for name in blob['names']:
        c = layer_case(blob, str(name))
        N, E = int(c['N']), len(c['src'])
        H, W, Wl, et = _case_tensors(G, c)
        rp, cs, ct = G.coo_to_csr(c['src'], c['dst'], et, N)
        out = G.layer_fwd(H, None, W, Wl, rp, cs, ct, G.d(c['ref_norm']), N, E, int(c['d_in']), int(c['d_out']),
                          int(c['nb']), bool(c['relu']))
        err = rel_err(out.cpu().numpy(), c['ref_out'])
        if str(name) in ('hand_kat', 'dup_edge', 'reverse'):
            assert err == 0.0, (name, err)          # small integers: exact in fp32
        assert err < TOL, (name, err)


def test_golden_layer_cases_backward(G):
    blob = load_npz('layer_cases.npz')
    for name in blob['names']:
        c = layer_case(blob, str(name))
        N, E = int(c['N']), len(c['src'])
        H, W, Wl, et = _case_tensors(G, c)
        rp, cs, ct = G.coo_to_csr(c['src'], c['dst'], et, N)
        norm = G.d(c['ref_norm'])
        out = G.layer_fwd(H, None, W, Wl, rp, cs, ct, norm, N, E, int(c['d_in']), int(c['d_out']), int(c['nb']),
                          bool(c['relu']))
        dH, dW, dWl = G.layer_bwd(H, None, W, Wl, c['src'], c['dst'], et, norm, out, G.d(c['G']), N, E,
                                  int(c['d_in']), int(c['d_out']), int(c['nb']), bool(c['relu']))
        assert rel_err(dH.cpu().numpy(), c['ref_dH']) < TOL, name
        assert rel_err(dW.cpu().numpy(), c['ref_dW']) < TOL, name
        if Wl is not None:
            assert rel_err(dWl.cpu().numpy(), c['ref_dWloop']) < TOL, name


def test_zero_edge_graph(G):
    blob = load_npz('layer_cases.npz')
    H, W, Wl = G.d(blob['zero_edge/H']), G.d(blob['zero_edge/W']), G.d(blob['zero_edge/Wloop'])
    rp = torch.zeros(5, dtype=torch.int32, device=G.DEV)
    norm = torch.ones(4, device=G.DEV)
    out = G.layer_fwd(H, None, W, Wl, rp, None, None, norm, 4, 0, 4, 4, 2, True)
    assert rel_err(out.cpu().numpy(), blob['zero_edge/ref_out']) < 1e-6


def test_empty_graph_and_bad_args(G):
    from renet_b200 import _lib
    L = _lib.lib()
    assert L.renet_rgcn_block_fwd(None, None, None, None, None, None, None, None, None, 0, 0, 200, 200, 100, 8, 1, None) == 0
    W = torch.zeros(8, 400, device=G.DEV)
    rc = L.renet_rgcn_block_fwd(_lib.ptr(W), None, _lib.ptr(W), None, None, None, None, None, None, 4, 3, 200, 200, 100, 8, 1, None)
    assert rc == -1


@pytest.fixture(scope='module')
def icews_batch():
    from renet_b200 import synthetic, utils
    tkg = synthetic.SyntheticTKG('icews18', seed=999, num_timestamps=40)
    q, sh, oh = tkg.batch(0, batch_size=1024, tail_only=True)
    hb = utils.assemble_history_batch_host(sh[0], sh[1], q[:, 0], tkg.graph_dict)
    return tkg, hb


def _oracle_layer(hb, H, W, Wl, et, relu):
    g = hb.graph
    dst = np.repeat(np.arange(len(g['node_ent'])), np.diff(g['row_ptr']))
    return restate.rgcn_block_layer(H, W, Wl, t(g['col_src']), t(dst), t(et.astype(np.int64)), t(g['norm']), relu, 100)


def test_icews18_shaped_batch_two_layers_vs_oracle(G, icews_batch):
    """Full-size ICEWS18-shaped history graph (about 11 k nodes / 33 k edges per 40-timestamp stream
    batch; the 240-timestamp bench shape is covered by the property tests below): both layers, the
    fused embedding lookup (h_index) included, against the CPU oracle on the same seeded inputs."""
    tkg, hb = icews_batch
    g = hb.graph
    N, E = len(g['node_ent']), len(g['col_src'])
    torch.manual_seed(0)
    ent = torch.randn(tkg.num_e, 200) * 0.1
    W1, W2 = torch.randn(512, 400) * 0.1, torch.randn(512, 400) * 0.1
    L1, L2 = torch.randn(200, 200) * 0.07, torch.randn(200, 200) * 0.07
    for reverse, et in ((False, g['col_type_s']), (True, g['col_type_o'])):
        H0 = ent[t(g['node_ent'])]
        o1 = _oracle_layer(hb, H0, W1, L1, et, True)
        o2 = _oracle_layer(hb, o1, W2, L2, et, False)
        rp, cs, ct = G.d(g['row_ptr'], torch.int32), G.d(g['col_src'], torch.int32), G.d(et, torch.int32)
        norm, idx = G.d(g['norm']), G.d(g['node_ent'], torch.int32)
        h1 = G.layer_fwd(ent.to(G.DEV), idx, W1.to(G.DEV), L1.to(G.DEV), rp, cs, ct, norm, N, E, 200, 200, 100, True)
        h2 = G.layer_fwd(h1, None, W2.to(G.DEV), L2.to(G.DEV), rp, cs, ct, norm, N, E, 200, 200, 100, False)
        assert rel_err(h1.cpu().numpy(), o1.numpy()) < TOL
        assert rel_err(h2.cpu().numpy(), o2.numpy()) < TOL


def test_module_autograd_vs_oracle(G, icews_batch):
    """RGCNBlockLayer modules (autograd.Function over the CUDA kernels) vs torch autograd on the oracle."""
    import torch.nn.functional as F
    from renet_b200 import utils
    from renet_b200.rgcn import RGCNBlockLayer
    tkg, hb_host = icews_batch
    import copy
    hb = utils.upload_history_batch(copy.copy(hb_host), torch.device(G.DEV))
    g = hb.graph
    gh = hb_host.graph if isinstance(hb_host.graph, dict) else None
    torch.manual_seed(1)
    ent = (torch.randn(tkg.num_e, 200) * 0.1)
    l1 = RGCNBlockLayer(200, 200, 512, 100, activation=F.relu, self_loop=True)
    l2 = RGCNBlockLayer(200, 200, 512, 100, activation=None, self_loop=True)
    Gout = torch.randn(g.N, 200)
    # oracle side
    P = [p.detach().clone().requires_grad_(True) for p in (ent, l1.weight, l1.loop_weight, l2.weight, l2.loop_weight)]
    node_ent = g.node_ent.cpu().long()
    dst = torch.repeat_interleave(torch.arange(g.N), (g.row_ptr[1:] - g.row_ptr[:-1]).cpu().long())
    src, et, norm = g.col_src.cpu().long(), g.col_type_s.cpu().long(), g.norm.cpu()
    o1 = restate.rgcn_block_layer(P[0][node_ent], P[1], P[2], src, dst, et, norm, True, 100)
    o2 = restate.rgcn_block_layer(o1, P[3], P[4], src, dst, et, norm, False, 100)
    (o2 * Gout).sum().backward()
    # CUDA side
    l1, l2 = l1.to(G.DEV), l2.to(G.DEV)
    ent_d = ent.to(G.DEV).requires_grad_(True)
    h1 = l1.apply_layer(g, ent_d, g.node_ent, False)
    h2 = l2.apply_layer(g, h1, None, False)
    assert rel_err(h2.detach().cpu().numpy(), o2.detach().numpy()) < TOL
    (h2 * Gout.to(G.DEV)).sum().backward()
    got = [ent_d.grad, l1.weight.grad, l1.loop_weight.grad, l2.weight.grad, l2.loop_weight.grad]
    for a, b, nm in zip(got, P, ('ent', 'W1', 'L1', 'W2', 'L2')):
        assert rel_err(a.cpu().numpy(), b.grad.numpy()) < TOL, nm


def test_full_size_properties(G):
    """Size-independent properties at the bench shape (N ~ 34 k, E ~ 200 k), no oracle needed:
    linearity in H without activation, invariance to the edge order inside the COO list, and
    agreement between host-built and device-built (renet_build_csr) CSR."""
    rng = np.random.RandomState(0)
    N, E, R2 = 34000, 200000, 512
    src, dst = rng.randint(0, N, E), (rng.zipf(1.3, E) % N)
    et = rng.randint(0, R2, E)
    deg = np.bincount(dst, minlength=N).astype(np.float32); deg[deg == 0] = 1
    norm = G.d(1.0 / deg)
    H = torch.randn(N, 200, device=G.DEV)
    W = torch.randn(R2, 400, device=G.DEV) * 0.1
    Wl = torch.randn(200, 200, device=G.DEV) * 0.07
    rp, cs, ct = G.coo_to_csr(src, dst, et, N)
    # device CSR == host CSR (stable)
    order = np.argsort(dst, kind='stable')
    np.testing.assert_array_equal(cs.cpu().numpy(), src[order])
    np.testing.assert_array_equal(ct.cpu().numpy(), et[order])
    np.testing.assert_array_equal(rp.cpu().numpy(), np.concatenate(([0], np.cumsum(np.bincount(dst, minlength=N)))))
    a = G.layer_fwd(H, None, W, Wl, rp, cs, ct, norm, N, E, 200, 200, 100, False)
    b = G.layer_fwd(H * 3.0, None, W, Wl, rp, cs, ct, norm, N, E, 200, 200, 100, False)
    assert rel_err(b.cpu().numpy(), (a * 3.0).cpu().numpy()) < 1e-5
    perm = rng.permutation(E)
    rp2, cs2, ct2 = G.coo_to_csr(src[perm], dst[perm], et[perm], N)
    c = G.layer_fwd(H, None, W, Wl, rp2, cs2, ct2, norm, N, E, 200, 200, 100, False)
    assert rel_err(c.cpu().numpy(), a.cpu().numpy()) < 1e-5
    # the gather hands partial sums between warps in a fixed order (no atomics): bitwise reproducible, so
    # relu(layer) == max(layer, 0) exactly and a second run gives the same bits
    r = G.layer_fwd(H, None, W, Wl, rp, cs, ct, norm, N, E, 200, 200, 100, True)
    assert torch.equal(r, torch.clamp_min(a, 0))
    assert torch.equal(G.layer_fwd(H, None, W, Wl, rp, cs, ct, norm, N, E, 200, 200, 100, False), a)


@pytest.mark.parametrize('N,E,heavy,empty_frac', [(5000, 40000, 6000, 0.25), (120, 20000, 0, 0.0), (40000, 17000, 0, 0.7),
                                                  (700000, 17000, 0, 0.9)])
def test_batch_scale_kernel_edge_cases_fwd_bwd_vs_oracle(G, N, E, heavy, empty_frac):
    """Whole-layer forward and backward against the CPU oracle on graphs with destinations without in-edges (also leading /
    trailing ones), a destination heavier than a whole CTA's share, far fewer destinations than warps and far more
    destinations than edges; the forward is bitwise reproducible.  With today's selection rule (gather_use_stream: E >= 16384
    and 2048 <= N <= 40960 for plain input rows, 16384 <= N for every backward) the four cases run:
      (5000, 40000)    forward on the persistent stream kernel (rgcn_stream.cuh), the 6 000-edge destination's chain of heads
                       included; dH on the tile kernel;
      (120, 20000)     tile kernels, forward and dH: 8 tiles of ~ 2 500 edges each;
      (40000, 17000)   stream kernel, forward and dH: about 300 destinations per CTA;
      (700000, 17000)  tile kernels, forward and dH: 43 750 tiles, most of them without an edge.
    The stream kernel's remaining paths (row_ptr read from global memory, every instantiation, the selection boundaries)
    are pinned per row, with the serving kernel asserted, in tests/rgcn_contract_check.py."""
    rng = np.random.RandomState(N + E)
    R2 = 480
    dst = rng.randint(0, N, E)
    if empty_frac:
        dead = rng.rand(N) < empty_frac
        dead[:7] = True; dead[-9:] = True
        alive = np.flatnonzero(~dead)
        dst = alive[rng.randint(0, len(alive), E)]
    if heavy:
        dst[:heavy] = alive[len(alive) // 2] if empty_frac else N // 2
    src, et = rng.randint(0, N, E), rng.randint(0, R2, E)
    deg = np.bincount(dst, minlength=N).astype(np.float32); deg[deg == 0] = 1
    norm = 1.0 / deg
    torch.manual_seed(0)
    H, W, Wl = torch.randn(N, 200) * 0.3, torch.randn(R2, 400) * 0.1, torch.randn(200, 200) * 0.07
    P = [p.clone().requires_grad_(True) for p in (H, W, Wl)]
    ref = restate.rgcn_block_layer(P[0], P[1], P[2], t(src), t(dst), t(et), t(norm), True, 100)
    # the upstream gradient is zeroed where the pre-activation is within 1e-4 of 0: there relu'(x) depends on the last bits
    # of x (3xTF32 GEMM vs CPU summation order), and one flipped element shifts gradients by far more than the tolerance
    with torch.no_grad():
        pre = restate.rgcn_block_layer(H, W, Wl, t(src), t(dst), t(et), t(norm), False, 100)
    Gout = torch.randn(ref.shape) * (pre.abs() > 1e-4)
    (ref * Gout).sum().backward()
    rp, cs, ct = G.coo_to_csr(src, dst, et, N)
    Hd, Wd, Wld, nd = H.to(G.DEV), W.to(G.DEV), Wl.to(G.DEV), G.d(norm)
    out = G.layer_fwd(Hd, None, Wd, Wld, rp, cs, ct, nd, N, E, 200, 200, 100, True)
    assert rel_err(out.cpu().numpy(), ref.detach().numpy()) < TOL
    assert torch.equal(out, G.layer_fwd(Hd, None, Wd, Wld, rp, cs, ct, nd, N, E, 200, 200, 100, True))
    dH, dW, dWl = G.layer_bwd(Hd, None, Wd, Wld, src, dst, et, nd, out, Gout.to(G.DEV), N, E, 200, 200, 100, True)
    assert rel_err(dH.cpu().numpy(), P[0].grad.numpy()) < TOL
    assert rel_err(dW.cpu().numpy(), P[1].grad.numpy()) < TOL
    assert rel_err(dWl.cpu().numpy(), P[2].grad.numpy()) < TOL


def test_hot_relation_list_only_changes_where_rows_are_read_from(G):
    """renet_rgcn_gather_hot: whatever relation ranking the caller passes (the true one, a wrong one, duplicates, a single id),
    the batch-scale kernel's output is bit-identical to renet_rgcn_gather's (which ranks per CTA) and to the tile kernel's
    within fp32 summation order."""
    from renet_b200 import _lib
    rng = np.random.RandomState(5)
    N, E, R2 = 30000, 150000, 480
    src = rng.randint(0, N, E)
    dst = rng.zipf(1.4, E) % N
    et = (rng.zipf(1.3, E) % R2).astype(np.int64)                  # skewed relation frequencies, as in the datasets
    deg = np.bincount(dst, minlength=N).astype(np.float32); deg[deg == 0] = 1
    rp, cs, ct = G.coo_to_csr(src, dst, et, N)
    torch.manual_seed(1)
    H = torch.randn(N, 200, device=G.DEV)
    W = torch.randn(R2, 400, device=G.DEV) * 0.1
    loop = torch.randn(N, 200, device=G.DEV)
    norm = G.d(1.0 / deg)
    L, P = _lib.lib(), _lib.ptr

    def run(hot):
        out = loop.clone()
        if hot is None:
            rc = L.renet_rgcn_gather(P(H), None, P(W), P(rp), P(cs), P(ct), P(norm), P(out), N, E, 200, 200, 100, R2, 1, 1, _lib.stream())
        else:
            h = G.d(np.asarray(hot, dtype=np.int32))
            rc = L.renet_rgcn_gather_hot(P(H), None, P(W), P(rp), P(cs), P(ct), P(norm), P(out), N, E, 200, 200, 100, R2, 1, 1,
                                         P(h), h.numel(), _lib.stream())
        _lib.check(rc, 'gather')
        return out

    base = run(None)
    freq = np.bincount(et, minlength=R2)
    for hot in (np.argsort(-freq)[:128], np.argsort(freq)[:40], [7, 7, 7, 3], [R2 - 1], np.arange(R2)[:200]):
        assert torch.equal(run(hot), base)
    ref = restate.rgcn_block_layer(H.cpu(), W.cpu(), None, t(src), t(dst), t(et), t(1.0 / deg), False, 100)
    assert rel_err(base.cpu().numpy(), torch.relu(ref + loop.cpu()).numpy()) < TOL
