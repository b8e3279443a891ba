"""-m gpu: programmatic dependent launch (RENET_PDL, DESIGN §4).  With PDL on, the RGCN step's chain (pack, dedup insert,
resident GEMM, dedup expand, stream gather) asks for the launch attribute, and every output is bitwise what plain stream
order (RENET_PDL=0) gives: a whole benchmark step on ICEWS18- and GDELT-shaped batches, the one-call inference encoder
(renet_encode_fwd) and a training step's loss and gradients, in normal and deterministic mode.  The host guard keeps the
plain order for a launch whose pre-wait inputs the previous launch writes."""
import contextlib
import os

import numpy as np
import pytest
import torch

from gpu_helpers import DEV, coo_to_csr
from renet_b200 import _lib

pytestmark = pytest.mark.gpu
H_DIM, NUM_BASES, BATCH = 200, 100, 1024


@contextlib.contextmanager
def pdl(on):
    before = os.environ.get('RENET_PDL')
    os.environ['RENET_PDL'] = '1' if on else '0'
    try:
        yield
    finally:
        if before is None:
            del os.environ['RENET_PDL']
        else:
            os.environ['RENET_PDL'] = before


# ---- the benchmark's device step (bench.py, region A) ------------------------------------------------------------------
_CASES = {}


def _case(workload):
    """bench.py's model and two pre-built batches of the workload (built once per module)"""
    if workload in _CASES:
        return _CASES[workload]
    from renet_b200 import hoststore, synthetic, utils
    from renet_b200.model import RENet
    tkg = synthetic.SyntheticTKG(workload, seed=999, h_dim=H_DIM)
    torch.manual_seed(999)
    model = RENet(tkg.num_e, H_DIM, tkg.num_r, dropout=0).to(DEV).eval()
    gstore = hoststore.GraphStore(tkg.graph_dict)
    pool = []
    for i in range(2):
        q, sh, oh = tkg.batch(i, BATCH, tail_only=False)
        dirs = []
        for hist, col, reverse in ((sh, 0, False), (oh, 2, True)):
            hb = utils.assemble_history_batch(hist[0], hist[1], q[:, col], tkg.graph_dict, DEV)
            g = hb.graph
            dirs.append({'g': g, 'reverse': reverse, 'ct': g.col_type(reverse), 'sub': g.readout_sub(hb.readout, reverse),
                         'S': hb.S})
        pool.append(dirs)
    _CASES[workload] = (model, 2 * tkg.num_r, gstore.hot_relations(DEV), pool)
    return _CASES[workload]


def _device_step(workload, dirs, step_no):
    """bench.py's device_step on fresh outputs: 2 directions x (layer 1 on the batched graph, layer 2 on the read-out
    sub-graph); returns ([h1, h2] per direction, library launches, PDL launches)"""
    model, R2, hot_rel, _ = _case(workload)
    L, P, stream = _lib.lib(), _lib.ptr, _lib.stream()
    agg = model.aggregator
    W1, L1, W2, L2 = (agg.rgcn1.weight.detach(), agg.rgcn1.loop_weight.detach(), agg.rgcn2.weight.detach(),
                      agg.rgcn2.loop_weight.detach())
    ent = model.ent_embeds.detach()
    outs = []
    torch.cuda.synchronize()
    n0, p0 = _lib.launch_count(), _lib.pdl_launch_count()
    L.renet_set_weight_generation(step_no)
    try:
        for d in dirs:
            g, sub, hot = d['g'], d['sub'], hot_rel[d['reverse']]
            h1 = torch.zeros(g.N, H_DIM, device=DEV)
            h2 = torch.zeros(d['S'], H_DIM, device=DEV)
            _lib.check(L.renet_selfloop_gemm(P(ent), P(g.node_ent), P(L1), P(h1), g.N, H_DIM, H_DIM, stream), 'gemm')
            _lib.check(L.renet_rgcn_gather_hot(P(ent), P(g.node_ent), P(W1), P(g.row_ptr), P(g.col_src), P(d['ct']), P(g.norm),
                                               P(h1), g.N, g.E, H_DIM, H_DIM, NUM_BASES, R2, 1, 1, P(hot), hot.numel(), stream),
                       'gather')
            _lib.check(L.renet_selfloop_gemm(P(h1), P(sub.uniq), P(L2), P(h2), sub.N, H_DIM, H_DIM, stream), 'gemm')
            _lib.check(L.renet_rgcn_gather_hot(P(h1), None, P(W2), P(sub.row_ptr), P(sub.col_src), P(sub.col_type(d['reverse'])),
                                               P(sub.norm), P(h2), sub.N, sub.E_cap, H_DIM, H_DIM, NUM_BASES, R2, 0, 1, P(hot),
                                               hot.numel(), stream), 'gather')
            outs += [h1, h2]
    finally:
        L.renet_set_weight_generation(-1)
    torch.cuda.synchronize()
    return outs, _lib.launch_count() - n0, _lib.pdl_launch_count() - p0


@pytest.mark.parametrize('workload', ['icews18', 'gdelt'])
def test_device_step_bitwise_and_chained(workload):
    pool = _case(workload)[3]
    for i, dirs in enumerate(pool):
        with pdl(False):
            ref, n_ref, p_ref = _device_step(workload, dirs, 10 * i + 1)
        with pdl(True):
            got, n_got, p_got = _device_step(workload, dirs, 10 * i + 2)
        assert p_ref == 0 and n_got == n_ref
        for k, (a, b) in enumerate(zip(ref, got)):
            assert torch.isfinite(a).all() and a.abs().sum() > 0, k
            assert torch.equal(a, b), 'output %d of batch %d differs' % (k, i)
        # DESIGN §4: the self-loop product (dedup insert -> resident GEMM -> expand from kDedupMinRows rows on, else the
        # resident GEMM alone), each self-loop weight packed once per step, and the stream gather where the dispatch picks
        # it (the tile kernel keeps plain launches): every launch of that chain asks for PDL
        assert p_got == _expected_pdl(dirs), (n_got, p_got, _expected_pdl(dirs))


def _expected_pdl(dirs):
    n = 2                                                           # the two packs
    for d in dirs:
        g, sub = d['g'], d['sub']
        n += 3 if g.N >= 16384 else 1                               # kDedupMinRows
        n += 3 if sub.N >= 16384 else 1
        n += int(g.E >= 16384 and 16384 <= g.N <= 40960)            # kStreamMinEdges, kStreamMinNodes, kStreamMaxNodes
        n += int(sub.E_cap >= 16384 and 2048 <= sub.N <= 40960)     # kStreamMinPlainNodes
    return n


def test_guard_keeps_plain_order_when_norm_aliases_the_previous_output():
    """A gather whose norm lies inside the rows the preceding self-loop product writes: the pre-wait inputs overlap the
    record, so the gather is launched without the attribute and its result equals plain order's.  Control: the same chain
    with a separate norm gets the attribute."""
    L, P, stream = _lib.lib(), _lib.ptr, _lib.stream()
    rng = np.random.RandomState(5)
    N, E, R2, T = 20000, 60000, 460, 23033
    src, dst, et = rng.randint(0, N, E), rng.randint(0, N, E), rng.randint(0, R2, E)
    rp, cs, ct = coo_to_csr(src, dst, et, N)
    g = torch.Generator(device=DEV).manual_seed(5)
    table = torch.randn(T, H_DIM, device=DEV, generator=g) * 0.5
    h_index = torch.randint(0, T, (N,), device=DEV, generator=g, dtype=torch.int32)
    W = torch.randn(R2, 400, device=DEV, generator=g) * 0.3
    Wl = torch.randn(H_DIM, H_DIM, device=DEV, generator=g) * 0.07
    own_norm = torch.rand(N, device=DEV, generator=g)

    def chain(aliased):
        prod = torch.empty(N, H_DIM, device=DEV)
        out = torch.empty(N, H_DIM, device=DEV)
        norm = prod.view(-1)[1000:1000 + N] if aliased else own_norm
        _lib.check(L.renet_selfloop_gemm(P(table), P(h_index), P(Wl), P(prod), N, H_DIM, H_DIM, stream), 'gemm')
        torch.cuda.synchronize()
        p0 = _lib.pdl_launch_count()
        _lib.check(L.renet_rgcn_gather(P(table), P(h_index), P(W), P(rp), P(cs), P(ct), P(norm), P(out), N, E, H_DIM, H_DIM,
                                       NUM_BASES, R2, 1, 0, stream), 'gather')
        torch.cuda.synchronize()
        return out, _lib.pdl_launch_count() - p0

    for aliased in (True, False):
        with pdl(False):
            ref, p_ref = chain(aliased)
        with pdl(True):
            got, p_got = chain(aliased)
        assert p_ref == 0
        assert p_got == (0 if aliased else 1), (aliased, p_got)
        assert torch.equal(ref, got), aliased


# ---- the inference encoder and the training step ----------------------------------------------------------------------
def _small_model():
    from renet_b200 import synthetic
    from renet_b200.model import RENet
    tkg = synthetic.SyntheticTKG('icews18', seed=3, h_dim=H_DIM)
    q, sh, oh = tkg.batch(3, batch_size=BATCH)
    torch.manual_seed(0)
    m = RENet(tkg.num_e, H_DIM, tkg.num_r, dropout=0).to(DEV)
    m.global_emb = tkg.global_emb
    return m, torch.from_numpy(q).long().to(DEV), sh, oh, tkg.graph_dict


def test_inference_encoder_bitwise():
    m, batch, sh, oh, gd = _small_model()
    m.eval()
    res = {}
    for on in (False, True):
        with pdl(on), torch.no_grad():
            p0 = _lib.pdl_launch_count()
            res[on] = [m(batch, sh, oh, gd, subject=s) for s in (True, False)]
            torch.cuda.synchronize()
            if on:
                assert _lib.pdl_launch_count() > p0
    for a, b in zip(res[False], res[True]):
        assert torch.isfinite(a).all() and torch.equal(a, b)


@pytest.mark.parametrize('det', [False, True])
def test_training_step_bitwise(det):
    """Deterministic mode: loss and every gradient bitwise.  Normal mode sums some gradients with float atomics, whose
    order changes from run to run in either mode: the loss is bitwise, the gradients agree to summation order."""
    m, batch, sh, oh, gd = _small_model()
    m.train()
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        res = {}
        for on in (False, True):
            m.zero_grad(set_to_none=True)
            with pdl(on):
                loss = m(batch, sh, oh, gd, subject=True)
                loss.backward()
                torch.cuda.synchronize()
            res[on] = [loss.detach().clone()] + [p.grad.clone() for p in m.parameters() if p.grad is not None]
    finally:
        torch.use_deterministic_algorithms(before)
        _lib.stream()
    assert len(res[False]) == len(res[True]) > 1
    for k, (a, b) in enumerate(zip(res[False], res[True])):
        if det or k == 0:
            assert torch.equal(a, b), k
        else:
            torch.testing.assert_close(b, a, rtol=1e-5, atol=1e-5 * float(a.abs().max()))
