"""-m gpu: RENet.evaluate_observed on the kernels.

* Against tests/golden/renet_eval_observed.npz (the reference's predict + encoder + linear per triple over its own history):
  ranks exact in all three protocols, loss to 1e-4.
* On the ICEWS18-shaped stream of test_gpu_eval_batched.py (three test timestamps) against a per-triple restatement on the
  GPU (_encode_one, ``linear``, the reference's rank rules) over a sample of triples: ranks exact except where a candidate's
  restated logit lies within 1e-6 of the label's (a measured tie, which may move the rank by at most the number of such
  candidates); those rows are counted and reported.
* Rank chunks forced small give the default's ranks bit for bit; encode budgets forced small (queries and components
  spanning chunk boundaries) give the default's encodings to 1e-5 of each row's max, and its ranks except for near ties.
* The test-time state and both RNG streams are unchanged.
* No logits are materialised (``linear.forward`` raises), and renet_decoder_rank_multi runs once per row chunk."""
import copy
import time

import numpy as np
import pytest
import torch

from helpers import eval_setup, load_npz, rel_err
from test_gpu_eval_batched import _icews18_stream

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def test_observed_kernels_match_reference_golden():
    from renet_b200 import _lib, synthetic
    ctx = eval_setup(DEV)
    m, quads, gold = ctx['model'], ctx['quads'], load_npz('renet_eval_observed.npz')
    S, ST, O, OT = ctx['hist']
    rows = gold['rows']
    gd = synthetic.build_graph_dict(quads, ctx['dims'][1])
    n0 = _lib.launch_count()
    out = m.evaluate_observed(quads[rows], ([S[i] for i in rows], [ST[i] for i in rows]), ([O[i] for i in rows], [OT[i] for i in rows]),
                              gd, dict(m.global_emb), total_data=quads, time_aware=True)
    assert _lib.launch_count() > n0
    for key, gk in (('raw', 'raw'), ('filtered', 'filt'), ('time_filtered', 'time_filt')):
        np.testing.assert_array_equal(out['protocols'][key]['ranks'], gold[gk].reshape(-1), err_msg=key)
    assert rel_err(out['loss'], float(gold['loss'].astype(np.float64).sum())) < 1e-4


def _split():
    quads, te, (S, ST, O, OT), ((m, _), (m_ref, _)) = _icews18_stream()
    args = (quads[te], ([S[i] for i in te], [ST[i] for i in te]), ([O[i] for i in te], [OT[i] for i in te]),
            dict(m.graph_dict), dict(m.global_emb))
    return quads, te, args, m, m_ref


def _restated_row(m, trip, hists, gd, ge):
    """(z_ob, z_sub) fp64 on the host for one triple: _encode_one over its own histories, then ``linear``."""
    R = m.num_rels
    s, r, o = (int(x) for x in trip[:3])
    sh, oh = hists
    with torch.no_grad():
        s_h = torch.zeros(m.h_dim, device=DEV) if len(sh[0]) == 0 else m._encode_one(s, r, sh[0], sh[1], True, gd, ge)
        o_h = torch.zeros(m.h_dim, device=DEV) if len(oh[0]) == 0 else m._encode_one(o, r, oh[0], oh[1], False, gd, ge)
        z_ob = m.linear(torch.cat((m.ent_embeds[s], s_h, m.rel_embeds[:R][r])))
        z_sub = m.linear(torch.cat((m.ent_embeds[o], o_h, m.rel_embeds[R:][r])))
    return z_ob.double().cpu().numpy(), z_sub.double().cpu().numpy()


def _rank(z, label, excluded):
    """The reference's rank rule (model.py:373-379, 403-418) on sigmoid scores with ``excluded`` zeroed (label kept), and
    the number of admissible candidates whose logit lies within 1e-6 max(1, |z|max) of the label's (a measured tie: the
    3xTF32 decoder against cuBLAS, and the batched encoding against _encode_one, differ by about that much)."""
    p = 1.0 / (1.0 + np.exp(-z))
    if excluded is not None:
        p = p.copy()
        p[excluded] = 0
        p[label] = 1.0 / (1.0 + np.exp(-z[label]))
    rank = (p > p[label]).sum() + ((p == p[label]).sum() - 1.0) / 2 + 1
    near = np.abs(z - z[label]) <= 1e-6 * max(1.0, float(np.abs(z).max()))
    near[label] = False
    if excluded is not None:
        near[excluded] = False
    return rank, int(near.sum())


def test_observed_kernels_match_per_triple_restatement_on_icews18_shape():
    quads, te, args, m, _ = _split()
    q, sh, oh, gd, ge = args
    out = m.evaluate_observed(*args, total_data=quads, time_aware=True)
    got = {k: out['protocols'][k]['ranks'].reshape(-1, 2) for k in ('raw', 'filtered', 'time_filtered')}
    sample = np.random.RandomState(3).choice(len(q), min(300, len(q)), replace=False)
    n_tie, n_rows, bad = 0, 0, []
    for i in sample:
        s, r, o, t = (int(x) for x in q[i])
        z_ob, z_sub = _restated_row(m, q[i], ((sh[0][i], sh[1][i]), (oh[0][i], oh[1][i])), gd, ge)
        same_t = quads[quads[:, 3] == t]
        for col, z, label, fix, fc, ans in ((1, z_ob, o, s, 0, 2), (0, z_sub, s, o, 2, 0)):
            excl = {'raw': None,
                    'filtered': quads[(quads[:, fc] == fix) & (quads[:, 1] == r), ans],
                    'time_filtered': same_t[(same_t[:, fc] == fix) & (same_t[:, 1] == r), ans]}
            for proto, ex in excl.items():
                ref, near = _rank(z, label, ex)
                n_rows += 1
                n_tie += near > 0
                g = got[proto][i, col]
                if abs(g - ref) > near:                       # a difference no measured tie accounts for
                    gap = np.sort(np.abs(z - z[label]))[1:4]
                    bad.append((int(i), proto, col, float(g), float(ref), near, gap.tolist()))
    print('evaluate_observed vs per-triple restatement: %d ranks, %d with a candidate within 1e-6 of the label '
          '(allowed to differ by at most that many places), %d unexplained differences %s' % (n_rows, n_tie, len(bad), bad[:10]))
    assert not bad
    assert n_tie <= n_rows // 2


def _captured_encodings(m, calls):
    """Wraps m._rank_triples to keep the s_h / o_h rows it is given (host copies), in call order."""
    orig = m._rank_triples

    def keep(quads, si, oi, s_h, o_h, *a, **k):
        calls.append((s_h.cpu(), o_h.cpu()))
        return orig(quads, si, oi, s_h, o_h, *a, **k)
    m._rank_triples = keep
    return orig


def test_observed_small_budgets_give_the_same_ranks(monkeypatch):
    """Rank chunks change nothing (a row's counts depend on that row alone): bitwise equal.  Encode chunks change which
    queries share a batched GEMM, so the encodings may differ in the last bits; they are compared row by row, and ranks may
    differ only where that flips a near tie."""
    from renet_b200 import inference
    quads, te, args, m, _ = _split()
    enc_ref = []
    orig = _captured_encodings(m, enc_ref)
    ref = m.evaluate_observed(*args, total_data=quads, time_aware=True)
    again = m.evaluate_observed(*args, total_data=quads, time_aware=True)
    monkeypatch.setattr(inference, 'OBSERVED_RANK_ROWS', 1000)
    rank_small = m.evaluate_observed(*args, total_data=quads, time_aware=True)
    for k in inference.PROTOCOLS:
        np.testing.assert_array_equal(again['protocols'][k]['ranks'], ref['protocols'][k]['ranks'], err_msg=k)
        np.testing.assert_array_equal(rank_small['protocols'][k]['ranks'], ref['protocols'][k]['ranks'], err_msg=k)
    assert rank_small['loss'] == ref['loss'] or rel_err(rank_small['loss'], ref['loss']) < 1e-6
    monkeypatch.setattr(inference, 'OBSERVED_RANK_ROWS', 16384)
    chunks = []
    enc = m.aggregator.encode
    m.aggregator.encode = lambda *a, **k: chunks.append(len(a[1])) or enc(*a, **k)
    monkeypatch.setattr(inference, 'ROLLOVER_SEQ_BUDGET', 300)
    monkeypatch.setattr(inference, 'EVAL_PLAN_BUDGET', 4000000)
    enc_small = []
    m._rank_triples = orig
    _captured_encodings(m, enc_small)
    got = m.evaluate_observed(*args, total_data=quads, time_aware=True)
    assert len(chunks) > 4, chunks                            # several encode chunks per direction
    worst = 0.0
    for a, b in zip(enc_ref[0], enc_small[0]):
        scale = a.abs().amax(dim=1, keepdim=True).clamp_min(1e-30)
        worst = max(worst, float(((a - b).abs() / scale).max()))
    n_diff = {}
    for k in inference.PROTOCOLS:
        d = np.abs(got['protocols'][k]['ranks'] - ref['protocols'][k]['ranks'])
        n_diff[k] = int((d > 0).sum())
        assert d.max() <= 2 and n_diff[k] <= len(d) // 200, (k, n_diff[k], d.max())
    print('small budgets: %d encode chunks of %s queries; encodings differ by at most %.2e of their row max; ranks that '
          'differ (near ties): %s of %d' % (len(chunks), chunks, worst, n_diff, len(ref['ranks'])))
    assert worst <= 1e-5
    assert rel_err(got['loss'], ref['loss']) < 1e-5


def test_observed_leaves_state_and_rng_unchanged():
    quads, te, args, m, _ = _split()
    keys = ('s_hist_test', 's_hist_test_t', 'o_hist_test', 'o_hist_test_t', 's_his_cache', 'o_his_cache', 's_his_cache_t',
            'o_his_cache_t')
    before = {k: copy.deepcopy(getattr(m, k)) for k in keys}
    latest = int(m.latest_time)
    gd_vals, ge_vals = list(m.graph_dict.items()), [(k, v.clone()) for k, v in m.global_emb.items()]
    torch.manual_seed(5)
    rng, cuda_rng = torch.get_rng_state(), torch.cuda.get_rng_state()
    m.evaluate_observed(*args, total_data=quads)
    assert torch.equal(torch.get_rng_state(), rng) and torch.equal(torch.cuda.get_rng_state(), cuda_rng)
    assert int(m.latest_time) == latest
    for k in keys:
        a, b = getattr(m, k), before[k]
        assert len(a) == len(b), k
        for x, y in zip(a, b):
            if isinstance(x, list):
                assert len(x) == len(y) and all(np.array_equal(np.asarray(u), np.asarray(v)) for u, v in zip(x, y)), k
            elif x is None or y is None:
                assert x is y, k
            else:
                assert np.array_equal(np.asarray(x), np.asarray(y)), k
    assert list(m.graph_dict.items()) == gd_vals
    assert [k for k, _ in ge_vals] == list(m.global_emb) and all(torch.equal(v, m.global_emb[k]) for k, v in ge_vals)


def test_observed_ranks_without_logits_once_per_row_chunk(monkeypatch):
    from renet_b200 import decoder, inference
    quads, te, args, m, _ = _split()
    ref = m.evaluate_observed(*args, total_data=quads, time_aware=True)

    def no_logits(*a, **k):
        raise AssertionError('linear.forward called: logits materialised')
    monkeypatch.setattr(m.linear, 'forward', no_logits)
    calls = []
    orig = decoder.decoder_rank_counts_multi

    def counted(x, *a, **k):
        calls.append(x.shape[0])
        return orig(x, *a, **k)
    monkeypatch.setattr(decoder, 'decoder_rank_counts_multi', counted)
    n, n_times = len(args[0]), len(np.unique(args[0][:, 3]))
    for rows in (inference.OBSERVED_RANK_ROWS, 2 * (n // 5 + 1)):
        monkeypatch.setattr(inference, 'OBSERVED_RANK_ROWS', rows)
        calls.clear()
        got = m.evaluate_observed(*args, total_data=quads, time_aware=True)
        per = rows // 2
        assert len(calls) == -(-n // per), (rows, calls)
        assert all(c <= rows for c in calls) and sum(calls) == 2 * n
        for k in inference.PROTOCOLS:
            np.testing.assert_array_equal(got['protocols'][k]['ranks'], ref['protocols'][k]['ranks'], err_msg=k)
        print('%d triples over %d timestamps: %d renet_decoder_rank_multi calls of %s rows' % (n, n_times, len(calls), calls))
    assert n_times == 3


def test_observed_call_time_is_reported():
    """Not a speed bar: the whole-split wall time at this shape, printed for the log (tools/bench_observed.py measures)."""
    quads, te, args, m, _ = _split()
    m.evaluate_observed(*args, total_data=quads)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    m.evaluate_observed(*args, total_data=quads)
    torch.cuda.synchronize()
    print('evaluate_observed: %d triples in %.1f ms' % (len(args[0]), (time.perf_counter() - t0) * 1e3))
