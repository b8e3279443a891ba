"""not gpu: histories longer than 16 steps on the host side -- the fp64 restatements against the reference's seq_len = 20
golden (tests/golden/renet_seq_len.npz, tools/gen_golden_seq_len.py), the C++ batcher and planner against the numpy
batcher at 17 to 64 steps, the test-time flow at seq_len = 20 (with the CPU oracle standing in for the CUDA encode, as in
test_inference_host.py), and the length-aware GRU workspace entries."""
import numpy as np
import pytest
import torch

from helpers import load_npz, rel_err
from oracle import restate

SEQ_LEN = 20


def _golden():
    return load_npz('renet_seq_len.npz')


def check_grad(g, tag, k, grad, tol=1e-4):
    """``grad`` against the golden's gradient of parameter k: whole, or its norm and marginals for a large matrix."""
    grad = np.asarray(grad, dtype=np.float64)
    if '%s/grad/%s' % (tag, k) in g:
        ref = g['%s/grad/%s' % (tag, k)]
        assert rel_err(grad, ref) < tol, (tag, k, rel_err(grad, ref))
        return True
    if '%s/grad_norm/%s' % (tag, k) in g:
        assert abs(np.linalg.norm(grad) - float(g['%s/grad_norm/%s' % (tag, k)])) < tol * float(g['%s/grad_norm/%s' % (tag, k)])
        for axis, name in ((1, 'rowsum'), (0, 'colsum')):
            ref = g['%s/grad_%s/%s' % (tag, name, k)]
            assert rel_err(grad.sum(axis), ref) < tol, (tag, k, name, rel_err(grad.sum(axis), ref))
        return True
    return False


def _params(shapes, seed, dtype=torch.float64):
    from oracle.gen_golden import det_params
    return {k: v.to(dtype).requires_grad_(True) for k, v in det_params(shapes, seed).items()}


def test_restated_forward_and_gradients_match_golden():
    from oracle.gen_golden import RENET_SHAPES, det_global_emb
    g = _golden()
    quads = g['quads'].astype(np.int64)
    num_e, R, h, nb, seed = int(g['num_e']), int(g['R']), int(g['h']), int(g['nb']), int(g['seed'])
    S, ST, O, OT = restate.build_history(quads, num_e, history_len=SEQ_LEN)
    sel = g['sel']
    np.testing.assert_array_equal([len(S[i]) for i in sel], g['sel_hist_len'])
    assert g['sel_hist_len'].max() == SEQ_LEN
    gd = restate.build_graph_dict(quads, R)
    glob = {t: v.double() for t, v in det_global_emb(np.unique(quads[:, 3]), h, seed + 1).items()}
    for subj, (H, HT) in ((True, (S, ST)), (False, (O, OT))):
        P = _params(RENET_SHAPES(num_e, h, R, nb), seed)
        out = restate.renet_forward(P, quads[sel], [H[i] for i in sel], [HT[i] for i in sel], gd, glob, subj, R, nb)
        out['loss'].backward()
        tag = 'subj' if subj else 'obj'
        assert abs(out['loss'].item() - float(g[tag + '/loss'])) < 1e-5 * abs(float(g[tag + '/loss']))
        assert len(out['batch_sizes']) == SEQ_LEN
        for k, p in P.items():
            if p.grad is not None:
                assert check_grad(g, tag, k, p.grad.numpy()), (tag, k, 'not in the golden')


@pytest.mark.parametrize('pool', [1, 0])
def test_restated_global_model_matches_golden(pool):
    from renet_b200.global_model import RENet_global
    g = _golden()
    quads = g['quads'].astype(np.int64)
    num_e, R, seed = int(g['num_e']), int(g['R']), int(g['seed'])
    times = np.unique(quads[:, 3])
    gd = restate.build_graph_dict(quads, R)
    shapes = {k: tuple(v.shape) for k, v in RENet_global(num_e, 200, R, seq_len=SEQ_LEN, maxpool=pool).state_dict().items()}
    sel = g['g_sel']
    for subj in (True, False):
        P = _params(shapes, seed + 5)
        loss = restate.global_forward(P, times[sel], g['true_prob_s'][sel], g['true_prob_o'][sel], gd, subj, maxpool=pool,
                                      seq_len=SEQ_LEN)
        loss.backward()
        tag = 'pool%d/%s' % (pool, 'subj' if subj else 'obj')
        assert abs(loss.item() - float(g[tag + '/loss'])) < 1e-5 * abs(float(g[tag + '/loss']))
        for k, p in P.items():
            if p.grad is not None:
                assert check_grad(g, tag, k, p.grad.numpy()), (tag, k, 'not in the golden')
    if pool == 1:
        # get_global_emb: the entry keyed by each timestamp is predict() at the next one (the last: one time unit on)
        P = {k: v.detach() for k, v in _params(shapes, seed + 5).items()}
        queries = list(times[1:]) + [times[-1] + (times[1] - times[0])]
        np.testing.assert_array_equal(g['global_emb_keys'], times)
        with torch.no_grad():
            emb = np.stack([restate.global_predict(P, int(t), gd, True, 1, SEQ_LEN)[0].numpy() for t in queries])
        assert rel_err(emb, g['global_emb']) < 1e-4


@pytest.mark.parametrize('length', [17, 20, 32, 64])
def test_host_batchers_equal_numpy_batcher_on_long_histories(length):
    from renet_b200 import synthetic, utils
    from renet_b200.hoststore import GraphStore, HistoryStore, assemble_view_raw, plan_view_raw, split_plan, split_raw
    quads, num_e, R = synthetic.make_quads('tiny', seed=5, num_timestamps=length + 30)
    S, ST, O, OT = synthetic.build_history(quads, history_len=length)
    gd = synthetic.build_graph_dict(quads, R)
    gs = GraphStore(gd)
    lens = np.asarray([len(x) for x in S])
    assert lens.max() == length
    rng = np.random.RandomState(length)
    sel = np.concatenate((np.flatnonzero(lens == length)[:40], rng.choice(len(quads), 200, replace=False)))
    store = HistoryStore(S, ST, quads[:, 0], gs)
    assert store.max_len == length
    view = store.select(sel)
    ref = utils.assemble_history_batch_host([S[i] for i in sel], [ST[i] for i in sel], quads[sel, 0], gd, sort=True)
    assert len(ref.batch_sizes) == length
    buf = np.zeros(1 << 22, dtype=np.int32)
    for raw, split in ((assemble_view_raw, split_raw), (plan_view_raw, split_plan)):
        r = raw(view, buf)
        np.testing.assert_array_equal(r['batch_sizes'], ref.batch_sizes)
        np.testing.assert_array_equal(r['s_idx'], ref.s_idx)
        parts = split(buf, r)
        np.testing.assert_array_equal(parts['seq_len'], ref.seq_len)
        np.testing.assert_array_equal(parts['seq_start'], np.concatenate(([0], np.cumsum(ref.seq_len)[:-1])))
        np.testing.assert_array_equal(parts['packed_row'], restate.packed_order(ref.seq_len)[0])
        np.testing.assert_array_equal(parts['node_ent'], ref.graph['node_ent'])
        np.testing.assert_array_equal(parts['readout'], ref.readout_host)
        if raw is assemble_view_raw:
            for k in ('row_ptr', 'col_src', 'col_type_s', 'col_type_o'):
                np.testing.assert_array_equal(parts[k], ref.graph[k])


def _eval_ctx():
    from oracle.gen_golden import RENET_SHAPES, det_global_emb, det_params
    from oracle.stub_global import StubGlobalModel
    from renet_b200 import synthetic
    from renet_b200.model import RENet
    from test_inference_host import _oracle_encode
    g = _golden()
    quads = g['quads'].astype(np.int64)
    num_e, R, h, nb, seed = int(g['num_e']), int(g['R']), int(g['h']), int(g['nb']), int(g['seed'])
    params = det_params(RENET_SHAPES(num_e, h, R, nb), seed)
    m = RENet(num_e, h, R, dropout=0, model=0, seq_len=SEQ_LEN, num_k=int(g['num_k']), num_bases=nb)
    m.load_state_dict(params, strict=True)
    m.eval()
    m.global_emb = det_global_emb(np.unique(quads[:, 3]), h, seed + 1)
    m.graph_dict = synthetic.build_graph_dict(quads, R)
    S, ST, O, OT = restate.build_history(quads, num_e, history_len=SEQ_LEN)
    pick = lambda L, idx: [L[i] for i in idx]                                           # noqa: E731
    tr, va, te = g['tr'], g['va'], g['te']
    m.init_history(quads[tr], (pick(S, tr), pick(ST, tr)), (pick(O, tr), pick(OT, tr)),
                   quads[va], (pick(S, va), pick(ST, va)), (pick(O, va), pick(OT, va)),
                   quads[te], (pick(S, te), pick(ST, te)), (pick(O, te), pick(OT, te)))
    ctx = dict(model=m, params=params, dims=(num_e, R, h, nb))
    m.aggregator.encode = _oracle_encode(ctx)
    m.latest_time = torch.tensor(int(g['t_test']))
    return m, g, quads, (S, ST, O, OT), StubGlobalModel(num_e, h, seed + 2)


def run_test_split(m, g, quads, hist, gm, batched):
    S, ST, O, OT = hist
    te = g['te']
    torch.manual_seed(4321)
    fn = m.evaluate_stream_batched if batched else m.evaluate_stream
    return fn(quads[te], ([S[i] for i in te], [ST[i] for i in te]), ([O[i] for i in te], [OT[i] for i in te]), gm,
              total_data=quads)


def check_rolled_histories(m, g):
    """The test-time histories after the roll-over equal the reference's; the golden guarantees one was trimmed at 20."""
    for side, hist_t in (('s', m.s_hist_test_t), ('o', m.o_hist_test_t)):
        np.testing.assert_array_equal([len(x) for x in hist_t], g['after_len_' + side])
        np.testing.assert_array_equal([list(x) + [-1] * (SEQ_LEN - len(x)) for x in hist_t], g['after_t_' + side])
    full = (g['before_len_s'] == SEQ_LEN) & (g['after_t_s'][:, -1] == int(g['t_test']))
    full |= (g['before_len_o'] == SEQ_LEN) & (g['after_t_o'][:, -1] == int(g['t_test']))
    assert full.any()


@pytest.mark.parametrize('batched', [False, True])
def test_test_time_flow_matches_golden(batched):
    m, g, quads, hist, gm = _eval_ctx()
    out = run_test_split(m, g, quads, hist, gm, batched)
    np.testing.assert_array_equal(out['ranks'], g['filt'].reshape(-1))
    assert abs(out['loss'] - float(g['loss'].sum())) < 1e-4 * float(g['loss'].sum())
    np.testing.assert_array_equal(np.asarray(gm.calls, dtype=np.int64), g['gm_calls'])
    check_rolled_histories(m, g)


def test_length_aware_workspace_entries():
    from renet_b200 import _lib
    L = _lib.lib()
    pairs = (('renet_gru_workspace_bytes', 'renet_gru_workspace_bytes_len'),
             ('renet_gru_bwd_workspace_bytes', 'renet_gru_bwd_workspace_bytes_len'),
             ('renet_gru_dropout_workspace_bytes', 'renet_gru_dropout_workspace_bytes_len'),
             ('renet_gru_bwd_dropout_workspace_bytes', 'renet_gru_bwd_dropout_workspace_bytes_len'))
    for S, Q, T, h in ((100, 10, 5, 200), (10240, 1024, 240, 200), (37, 3, 1, 8)):
        for old, new in pairs:
            assert hasattr(L, new)
            base = getattr(L, old)(S, Q, T, h)
            for n in (0, 1, 10, 16):
                assert getattr(L, new)(S, Q, T, h, n) == base, (old, n)
            prev = base
            for n in (17, 20, 32, 64, 80):
                cur = getattr(L, new)(S, Q, T, h, n)
                assert cur > prev, (new, n)
                prev = cur
            # per step above 16: GH + Hs (8h floats per sequence) forward, dGH (6h) backward
            per_step = (8 if 'bwd' not in new else 6) * h * Q * 4
            assert abs(getattr(L, new)(S, Q, T, h, 32) - base - 16 * per_step) <= 64, new
