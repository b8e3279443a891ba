"""-m gpu: RENet.forecast_observed on the kernels.

* Against tests/golden/renet_eval_observed.npz (the reference's scores per triple over its own history), with the histories
  built from the facts by synthetic.observed_history: top-k ids, values and known answers left out, in both directions.
* On the ICEWS18-shaped stream of test_gpu_eval_observed.py against a per-query restatement (_encode_one, ``linear`` in
  fp64 with cuBLAS, softmax, the known answers taken out) on a few hundred sampled queries, both directions, static and
  time-aware: id sets exact outside the near-tie band of the restatement's logits, inside it every returned logit within
  the band of the k-th; values to 1e-3 relative.  The band count is printed: the untrained test model's logits crowd
  together (DESIGN section 5, observed evaluation).
* Row chunks forced small give the default's result bit for bit; encode budgets forced small give its id sets outside
  the near-tie band.
* One renet_decoder_topk call per row chunk and no logits (``linear.forward`` raises); the test-time state and both RNG
  streams are unchanged."""
import copy

import numpy as np
import pytest
import torch

from helpers import eval_setup, load_npz
from test_forecast_observed_host import _allowed, _queries, check_against_scores
from test_gpu_eval_observed import _split

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def test_forecast_observed_kernels_match_reference_golden():
    from renet_b200 import _lib, synthetic
    ctx = eval_setup(DEV)
    m, quads = ctx['model'], ctx['quads']
    ctx['gold'] = gold = load_npz('renet_eval_observed.npz')
    gd, ge = synthetic.build_graph_dict(quads, ctx['dims'][1]), dict(m.global_emb)
    n0 = _lib.launch_count()
    bands = {}
    for subject in (True, False):
        z = (gold['ob_pred'] if subject else gold['sub_pred']).astype(np.float64)
        q, hist = _queries(ctx, subject)
        for case, known in (('none', None), ('static', quads[:, :3]), ('time_aware', quads)):
            for k in (5, m.in_dim):
                vals, ids = m.forecast_observed(q, hist, gd, ge, k=k, subject=subject, known=known,
                                                time_aware=case == 'time_aware')
                assert vals.is_cuda and ids.is_cuda and vals.dtype == torch.float32 and ids.dtype == torch.long
                allowed = _allowed(quads, q, subject, case, m.in_dim)
                bands[(subject, case, k)] = check_against_scores(vals, ids, z, allowed, k, 1e-5, 1e-5)
    assert _lib.launch_count() > n0
    print('golden: rows in the near-tie band per (subject, filter, k): %s' % bands)
    assert max(bands.values()) <= len(gold['rows']) // 10


def _direction(args, quads, subject):
    """(queries, history) of one direction of the split."""
    q, sh, oh = args[:3]
    c = 0 if subject else 2
    return np.stack((q[:, c], q[:, 1], q[:, 3]), 1), (sh if subject else oh)


def _restated_logits(m, queries, hist, rows, subject, gd, ge):
    """z fp64 [len(rows), N]: _encode_one over each query's own history (zero when empty), then ``linear`` in fp64."""
    R = m.num_rels
    rel = m.rel_embeds[:R] if subject else m.rel_embeds[R:]
    W, b = m.linear.weight.double(), m.linear.bias.double()
    out = []
    with torch.no_grad():
        for i in rows:
            e, r, _ = (int(x) for x in queries[i])
            hl, ht = hist[0][i], hist[1][i]
            s_h = torch.zeros(m.h_dim, device=DEV) if len(hl) == 0 else m._encode_one(e, r, hl, ht, subject, gd, ge)
            x = torch.cat((m.ent_embeds[e], s_h, rel[r])).double()
            out.append((W @ x + b).cpu())
    return torch.stack(out).numpy()


@pytest.mark.parametrize('subject', [True, False])
def test_forecast_observed_matches_per_query_restatement_on_icews18_shape(subject):
    quads, te, args, m, _ = _split()
    gd, ge = args[3], args[4]
    queries, hist = _direction(args, quads, subject)
    k = 10
    rows = np.sort(np.random.RandomState(4).choice(len(queries), min(300, len(queries)), replace=False))
    z = _restated_logits(m, queries, hist, rows, subject, gd, ge)
    eps = 1e-5 * max(1.0, float(np.abs(z).max()))          # cuBLAS fp64 against 3xTF32 logits, and s_h to ~1e-6
    for case, known in (('static', quads[:, :3]), ('time_aware', quads)):
        vals, ids = m.forecast_observed(queries, hist, gd, ge, k=k, subject=subject, known=known,
                                        time_aware=case == 'time_aware')
        allowed = _allowed(quads, queries[rows], subject, case, m.in_dim)
        n_band = check_against_scores(vals[rows], ids[rows], z, allowed, k, eps, 1e-3, relative=True)
        print('forecast_observed vs restatement (%s, %s): %d rows, %d in the near-tie band of %.2e'
              % ('objects' if subject else 'subjects', case, len(rows), n_band, eps))


def test_small_row_chunks_and_encode_budgets(monkeypatch):
    """Row chunks change nothing (a row's top-k depends on that row alone): bitwise equal.  Encode chunks change which
    queries share a batched GEMM, so the values may move in the last bits; the id sets must agree wherever the k-th and
    (k+1)-th values are further apart than that."""
    from renet_b200 import inference
    quads, te, args, m, _ = _split()
    gd, ge = args[3], args[4]
    queries, hist = _direction(args, quads, False)
    k = 10

    def run():
        return m.forecast_observed(queries, hist, gd, ge, k=k + 1, subject=False, known=quads, time_aware=True)
    ref = run()
    for rows in (1000, 7):
        monkeypatch.setattr(inference, 'OBSERVED_RANK_ROWS', rows)
        got = run()
        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]), rows
    monkeypatch.setattr(inference, 'OBSERVED_RANK_ROWS', 16384)
    chunks = []
    enc = m.aggregator.encode
    monkeypatch.setattr(m.aggregator, 'encode', lambda *a, **kw: chunks.append(len(a[1])) or enc(*a, **kw))
    monkeypatch.setattr(inference, 'ROLLOVER_SEQ_BUDGET', 300)
    monkeypatch.setattr(inference, 'EVAL_PLAN_BUDGET', 4000000)
    vals, ids = run()
    assert len(chunks) > 4, chunks
    rv, ri, gi = ref[0].cpu().double().numpy(), ref[1].cpu().numpy(), ids.cpu().numpy()
    clear = rv[:, k - 1] - rv[:, k] > 1e-5 * rv[:, k - 1]
    for j in np.flatnonzero(clear):
        assert set(gi[j, :k].tolist()) == set(ri[j, :k].tolist()), j
    worst = float(np.abs(vals.cpu().double().numpy() - rv).max() / rv.max())
    print('small budgets: %d encode chunks; %d of %d rows outside the near-tie band, id sets equal there; values moved by '
          'at most %.2e of the largest' % (len(chunks), int(clear.sum()), len(rv), worst))
    assert clear.sum() >= len(rv) // 2


def test_one_topk_call_per_row_chunk_and_no_logits(monkeypatch):
    from renet_b200 import decoder, inference
    quads, te, args, m, _ = _split()
    gd, ge = args[3], args[4]
    queries, hist = _direction(args, quads, True)
    n = len(queries)
    ref = m.forecast_observed(queries, hist, gd, ge, k=10, known=quads[:, :3])

    def no_logits(*a, **kw):
        raise AssertionError('linear.forward called: logits materialised')
    monkeypatch.setattr(m.linear, 'forward', no_logits)
    calls = []
    orig = decoder.decoder_topk

    def counted(x, *a, **kw):
        calls.append(x.shape[0])
        out = orig(x, *a, **kw)
        assert out[0].shape == (x.shape[0], 10)
        return out
    monkeypatch.setattr(decoder, 'decoder_topk', counted)
    for rows in (inference.OBSERVED_RANK_ROWS, n // 5 + 1):
        monkeypatch.setattr(inference, 'OBSERVED_RANK_ROWS', rows)
        calls.clear()
        got = m.forecast_observed(queries, hist, gd, ge, k=10, known=quads[:, :3])
        assert len(calls) == -(-n // rows) and all(c <= rows for c in calls) and sum(calls) == n, (rows, calls)
        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
        print('%d queries: %d renet_decoder_topk calls of %s rows' % (n, len(calls), calls))


def test_forecast_observed_leaves_state_and_rng_unchanged():
    quads, te, args, m, _ = _split()
    gd, ge = args[3], args[4]
    keys = ('s_hist_test', 's_hist_test_t', 'o_hist_test', 'o_hist_test_t', 's_his_cache', 'o_his_cache', 's_his_cache_t',
            'o_his_cache_t')
    before = {k: copy.deepcopy(getattr(m, k)) for k in keys}
    latest = int(m.latest_time)
    gd_vals, ge_vals = list(m.graph_dict.items()), [(k, v.clone()) for k, v in m.global_emb.items()]
    torch.manual_seed(5)
    rng, cuda_rng = torch.get_rng_state(), torch.cuda.get_rng_state()
    for subject in (True, False):
        m.forecast_observed(*_direction(args, quads, subject), gd, ge, k=10, subject=subject, known=quads, time_aware=True)
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
