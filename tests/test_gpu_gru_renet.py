"""-m gpu: fused read-out + GRU and the whole RENet.forward against the reference goldens / CPU oracle."""
import numpy as np
import pytest
import torch

from helpers import load_npz, rel_err
from oracle import restate
from oracle.gen_golden import RENET_SHAPES, det_global_emb, det_params

pytestmark = pytest.mark.gpu
TOL = 1e-4
DEV = 'cuda:0'


def _setup(fname):
    from renet_b200 import synthetic
    from renet_b200.model import RENet
    b = load_npz(fname)
    quads = b['quads'].astype(np.int64)
    num_e, R, h, nb, seed = int(b['num_e']), int(b['R']), int(b['h']), int(b['nb']), int(b['seed'])
    params = det_params(RENET_SHAPES(num_e, h, R, nb), seed)
    m = RENet(num_e, h, R, dropout=0, model=0, seq_len=10, num_k=10, num_bases=nb)
    m.load_state_dict(params, strict=True)          # reference state_dict keys load as is
    m = m.to(DEV)
    glob = det_global_emb(np.unique(quads[:, 3]), h, seed + 1)
    m.global_emb = glob
    gd = synthetic.build_graph_dict(quads, R)
    S, ST, O, OT = synthetic.build_history(quads)
    sel = b['sel']
    pick = lambda lst: [lst[i] for i in sel]
    batch = torch.from_numpy(quads[sel]).long().to(DEV)
    return b, m, params, glob, gd, batch, (pick(S), pick(ST)), (pick(O), pick(OT)), quads, sel, (num_e, R, h, nb)


@pytest.mark.parametrize('fname', ['renet_tiny.npz', 'renet_icews18_slice.npz'])
def test_renet_forward_matches_reference_golden(fname):
    b, m, params, glob, gd, batch, sh, oh, quads, sel, dims = _setup(fname)
    m.eval()
    for tag, subj in (('subj', True), ('obj', False)):
        with torch.no_grad():
            s, r, o, s_h, s_q, rel = m.encode(batch, sh, oh, gd, subject=subj)
            loss = m.decode_loss(s, r, o, s_h, s_q, rel)
        ref_loss = float(b[tag + '/loss'])
        assert abs(loss.item() - ref_loss) < TOL * abs(ref_loss), (tag, loss.item(), ref_loss)
        Q = b[tag + '/s_h'].shape[0]
        # ties among equal history lengths may be ordered differently (reference sort is unstable)
        for got, ref in ((s_h[:Q], b[tag + '/s_h']), (s_q[:Q], b[tag + '/s_q'])):
            assert rel_err(np.sort(got.cpu().numpy(), axis=0), np.sort(ref, axis=0)) < TOL
        assert torch.count_nonzero(s_h[Q:]) == 0


@pytest.mark.parametrize('fname', ['renet_tiny.npz', 'renet_icews18_slice.npz'])
def test_aggregator_packed_inputs_match_reference_golden(fname):
    """RGCNAggregator.forward returns the reference's two PackedSequences (Aggregator.py:160-165)."""
    b, m, params, glob, gd, batch, sh, oh, quads, sel, (num_e, R, h, nb) = _setup(fname)
    m.eval()
    for tag, subj, hist in (('subj', True, sh), ('obj', False, oh)):
        rel = m.rel_embeds[:R] if subj else m.rel_embeds[R:]
        s = batch[:, 0] if subj else batch[:, 2]
        with torch.no_grad():
            p4, p3 = m.aggregator(hist, s, batch[:, 1], m.ent_embeds, rel, gd, glob, reverse=not subj)
        np.testing.assert_array_equal(p4.batch_sizes.numpy(), b[tag + '/batch_sizes'])
        assert p4.data.shape[1] == 4 * h and p3.data.shape[1] == 3 * h
        assert rel_err(p4.data.double().sum(0).cpu().numpy(), b[tag + '/x4_sum']) < TOL
        assert rel_err(p3.data.double().sum(0).cpu().numpy(), b[tag + '/x3_sum']) < TOL


def test_training_path_gradients_match_reference_golden():
    """loss.backward() through the CUDA kernels (unfused GRU modules) vs the reference's gradients."""
    fname = 'renet_tiny.npz'
    b, m, params, glob, gd, batch, sh, oh, quads, sel, dims = _setup(fname)
    m.train()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    for tag, subj in (('subj', True), ('obj', False)):
        m.zero_grad()
        loss = m.forward_unfused(batch, sh, oh, gd, subject=subj)
        loss.backward()
        assert abs(loss.item() - float(b[tag + '/loss'])) < TOL * abs(float(b[tag + '/loss']))
        for k, p in m.named_parameters():
            key = tag + '/grad/' + k
            if key in b.files:
                assert rel_err(p.grad.cpu().numpy(), b[key]) < 5 * TOL, (tag, k)


@pytest.mark.parametrize('fname', ['renet_tiny.npz', 'renet_icews18_slice.npz'])
def test_fused_training_step_gradients_match_reference_golden(fname):
    """RENet.forward (fused RGCN + fused GRU, dropout 0) -> loss.backward() entirely through the CUDA
    kernels (renet_rgcn_block_bwd, renet_gru_bwd) vs the reference's autograd gradients."""
    b, m, params, glob, gd, batch, sh, oh, quads, sel, dims = _setup(fname)
    m.train()
    for tag, subj in (('subj', True), ('obj', False)):
        m.zero_grad()
        loss = m(batch, sh, oh, gd, subject=subj)
        loss.backward()
        assert abs(loss.item() - float(b[tag + '/loss'])) < TOL * abs(float(b[tag + '/loss']))
        for k, p in m.named_parameters():
            if (tag + '/grad/' + k) in b.files:
                assert rel_err(p.grad.cpu().numpy(), b[tag + '/grad/' + k]) < 5 * TOL, (tag, k)
            else:
                g = p.grad.double().cpu()
                scale = float(b['%s/grad_norm/%s' % (tag, k)])
                assert abs(g.norm().item() - scale) < 5 * TOL * scale, (tag, k)
                for ax, nm in ((1, 'grad_rowsum'), (0, 'grad_colsum')):
                    diff = np.abs(g.sum(ax).numpy() - b['%s/%s/%s' % (tag, nm, k)]).max()
                    assert diff < 50 * TOL * scale, (tag, k, nm)


def test_fused_gru_vs_oracle_synthetic():
    """renet_gru_fwd on an ICEWS18-shaped batch (h=200) against the CPU oracle's explicit recurrence."""
    from renet_b200 import synthetic, utils
    from renet_b200.gru import fused_gru
    tkg = synthetic.SyntheticTKG('icews18', seed=3, num_timestamps=24)
    q, sh, oh = tkg.batch(0, batch_size=512)
    hb = utils.assemble_history_batch(sh[0], sh[1], q[:, 0], tkg.graph_dict, torch.device(DEV))
    torch.manual_seed(0)
    h = 200
    N = hb.graph.N
    H2 = torch.randn(N, h) * 0.5
    ent, rel = torch.randn(tkg.num_e, h) * 0.3, torch.randn(tkg.num_r, h) * 0.3
    glob = torch.randn(len(hb.times), h) * 0.1
    enc, enc_r = torch.nn.GRU(4 * h, h, batch_first=True), torch.nn.GRU(3 * h, h, batch_first=True)
    s_tem = torch.from_numpy(q[:, 0][hb.s_idx])
    r_tem = torch.from_numpy(q[:, 1][hb.s_idx])
    Q = hb.num_seq
    X4, X3, perm, bs = restate.packed_inputs(H2, hb.readout.cpu().long(), hb.seq_len, s_tem, r_tem, ent, rel,
                                             glob[hb.row_glob.cpu().long()])
    with torch.no_grad():
        ref4 = restate.gru_final_hidden_batched(X4, hb.seq_len, enc.weight_ih_l0, enc.weight_hh_l0, enc.bias_ih_l0, enc.bias_hh_l0)
        ref3 = restate.gru_final_hidden_batched(X3, hb.seq_len, enc_r.weight_ih_l0, enc_r.weight_hh_l0, enc_r.bias_ih_l0, enc_r.bias_hh_l0)
        enc, enc_r = enc.to(DEV), enc_r.to(DEV)
        hn4, hn3 = fused_gru(H2.to(DEV), ent.to(DEV), rel.to(DEV), glob.to(DEV), hb,
                             s_tem[:Q].to(torch.int32).to(DEV), r_tem[:Q].to(torch.int32).to(DEV), enc, enc_r)
    assert rel_err(hn4.cpu().numpy(), ref4.numpy()) < TOL
    assert rel_err(hn3.cpu().numpy(), ref3.numpy()) < TOL


def test_no_cpu_fallback():
    from renet_b200.rgcn import RGCNBlockLayer
    from renet_b200 import _lib
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        _lib.require_cuda(torch.zeros(3))
    assert _lib.launch_count() > 0


def test_cpp_batcher_path_equals_list_path():
    """RENet.encode fed with HistoryViews (flat stores + C++ batcher) == fed with the reference's lists."""
    from renet_b200 import hoststore
    b, m, params, glob, gd, batch, sh, oh, quads, sel, (num_e, R, h, nb) = _setup('renet_icews18_slice.npz')
    from renet_b200 import synthetic
    S, ST, O, OT = synthetic.build_history(quads)
    gs = hoststore.GraphStore(gd)
    vs = hoststore.HistoryStore(S, ST, quads[:, 0], gs).select(sel)
    vo = hoststore.HistoryStore(O, OT, quads[:, 2], gs).select(sel)
    m.eval()
    with torch.no_grad():
        for subj in (True, False):
            a = m.encode(batch, sh, oh, gd, subject=subj)
            c = m.encode(batch, vs, vo, gs, subject=subj)
            for x, y in zip(a[:5], c[:5]):
                assert torch.allclose(x.float(), y.float(), atol=1e-5)


def test_prefetched_batches_equal_direct_assembly():
    """hoststore.prefetch (worker threads + pinned staging ring) yields the same device batches as assemble_view."""
    from renet_b200 import hoststore, synthetic
    tkg = synthetic.SyntheticTKG('icews18', seed=4, num_timestamps=16)
    gs = hoststore.GraphStore(tkg.graph_dict)
    hs = hoststore.HistoryStore(tkg.s_hist, tkg.s_hist_t, tkg.quads[:, 0], gs)
    sels = [tkg.batch_indices(i, 256) for i in range(5)]
    dev = torch.device(DEV)
    got = list(hoststore.prefetch(((hs.select(s),) for s in sels), dev, depth=2, workers=2))
    assert len(got) == 5
    for (hb,), s in zip(got, sels):
        ref = hoststore.assemble_view(hs.select(s), dev)
        assert hb.graph.E == ref.graph.E        # device batcher: resolves the asynchronous edge count (and trims col_*)
        for name in ('node_ent', 'row_ptr', 'col_src', 'col_type_s', 'col_type_o', 'norm'):
            assert torch.equal(getattr(hb.graph, name), getattr(ref.graph, name)), name
        assert torch.equal(hb.readout, ref.readout) and torch.equal(hb.packed_row, ref.packed_row)
        np.testing.assert_array_equal(hb.s_idx, ref.s_idx)
        np.testing.assert_array_equal(hb.batch_sizes, ref.batch_sizes)


def test_packed_weight_cache_tracks_in_place_updates():
    """The tensor-core engine caches packed weights per (module, addresses, in-place versions): repeated encodes reuse the
    images, an in-place update (what an optimiser step is) re-packs, and the result equals a fresh module's."""
    import copy
    from renet_b200 import _lib
    b, m, params, glob, gd, batch, sh, oh, quads, sel, dims = _setup('renet_icews18_slice.npz')
    m.eval()

    def run(model):
        with torch.no_grad():
            return [torch.cat(model.encode(batch, sh, oh, gd, subject=subj)[3:5], 1).clone() for subj in (True, False)]
    n0 = _lib.launch_count()
    a1 = run(m)
    n1 = _lib.launch_count()
    a2 = run(m)
    n2 = _lib.launch_count()
    assert all(torch.equal(x, y) for x, y in zip(a1, a2))
    assert n2 - n1 < n1 - n0                                   # the second pass skipped the packing launches
    with torch.no_grad():
        m.encoder.weight_hh_l0.mul_(1.25)
        m.aggregator.rgcn2.loop_weight.add_(0.01)
    a3 = run(m)
    assert not torch.equal(a3[0], a1[0])
    fresh = copy.deepcopy(m)
    fresh.aggregator._pack_token = _lib.new_pack_token()
    fresh.global_emb = m.global_emb
    a4 = run(fresh)
    assert all(torch.equal(x, y) for x, y in zip(a3, a4))
