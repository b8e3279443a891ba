"""not gpu: RENet.forecast_observed and synthetic.observed_history (renet_b200/inference.py, synthetic.py) with the model on the
host, the CPU oracle standing in for the CUDA encode as in test_eval_observed_host.py.

* Against tests/golden/renet_eval_observed.npz (the unmodified reference's scores per triple over its own history), with
  the histories built from the facts by observed_history: the ids are the golden scores' top-k (ties to the lower id), the
  values their softmax, and the known answers are left out, statically and time-aware.
* With no filter and k = every entity, each triple's answer sits at evaluate_observed's raw rank.
* observed_history equals build_history (the product's and the oracle's) for every quadruple of two streams, shares one
  array per (entity, timestamp), and a window holds only timestamps strictly before its query's.
* Row chunks forced small, and the queries permuted, give the same rows bit for bit.
* The test-time state, torch's RNG and the module's mode are unchanged; every argument error comes before any work."""
import copy

import numpy as np
import pytest
import torch

from test_eval_observed_host import STATE, _ctx, _same

from oracle import restate
from renet_b200 import synthetic


def _queries(ctx, subject, rows=None):
    """The golden's triples as queries of one direction, with their histories built from every known quadruple."""
    quads = ctx['quads']
    q = quads[ctx['gold']['rows'] if rows is None else rows]
    c = 0 if subject else 2
    return np.stack((q[:, c], q[:, 1], q[:, 3]), 1), synthetic.observed_history(quads, q[:, c], q[:, 3], subject)


def _forecast(ctx, subject, k, known=None, time_aware=False, rows=None):
    q, hist = _queries(ctx, subject, rows)
    return ctx['model'].forecast_observed(q, hist, ctx['gd'], ctx['ge'], k=k, subject=subject, known=known,
                                          time_aware=time_aware)


def _allowed(quads, q, subject, case, num_e):
    """bool [n, num_e]: the answers each query may return -- all, or all but those known for (e, r) (case 'static') or for
    (e, r, t) ('time_aware'), found by scanning the quadruples."""
    fix, ans = (0, 2) if subject else (2, 0)
    out = np.ones((len(q), num_e), dtype=bool)
    if case != 'none':
        for i, (e, r, t) in enumerate(q):
            sel = (quads[:, fix] == e) & (quads[:, 1] == r)
            if case == 'time_aware':
                sel &= quads[:, 3] == t
            out[i, quads[sel, ans]] = False
    return out


def check_against_scores(vals, ids, z, allowed, k, band, vtol, relative=False):
    """forecast's contract against reference scores z [n, N] (fp64): per row the admissible ids by z descending, ties to the
    lower id, then -1 / 0.  Where the k-th and (k+1)-th admissible scores differ by more than ``band`` the id set is exact,
    and so is the order where no two neighbours of the top k lie within ``band``; otherwise (the near-tie band) every
    returned score lies within ``band`` of the k-th.  Always distinct admissible ids, descending within ``band``.  Values
    equal softmax(z) over all N within ``vtol`` (of the value with ``relative``).  Returns the number of rows in the band."""
    vals, ids = vals.cpu().double().numpy(), ids.cpu().numpy()
    assert vals.shape == ids.shape == (len(z), k)
    n_band = 0
    for m in range(len(z)):
        adm = np.flatnonzero(allowed[m])
        order = adm[np.argsort(-z[m, adm], kind='stable')]
        kk = min(k, len(adm))
        assert (ids[m, kk:] == -1).all() and (vals[m, kk:] == 0).all(), m
        if kk == 0:
            continue
        got = ids[m, :kk]
        assert (got >= 0).all() and allowed[m][got].all() and len(set(got.tolist())) == kk, m
        assert (np.diff(z[m, got]) <= band).all(), m
        zs = z[m, order[:kk + 1]]
        if kk < len(adm) and zs[kk - 1] - zs[kk] <= band:
            n_band += 1
            assert z[m, got].min() >= zs[kk - 1] - band, m
        elif kk > 1 and np.diff(zs[:kk]).max() >= -band:
            assert set(got.tolist()) == set(order[:kk].tolist()), m
        else:
            np.testing.assert_array_equal(got, order[:kk], err_msg=str(m))
        p = np.exp(z[m] - z[m].max())
        p = p[got] / p.sum()
        err = np.abs(vals[m, :kk] - p) / (p if relative else 1.0)
        assert err.max() <= vtol, (m, err.max())
    return n_band


@pytest.mark.parametrize('case', ['none', 'static', 'time_aware'])
@pytest.mark.parametrize('subject', [True, False])
def test_forecast_observed_matches_reference_golden(subject, case):
    ctx = _ctx()
    quads, gold, num_e = ctx['quads'], ctx['gold'], ctx['dims'][0]
    z = (gold['ob_pred'] if subject else gold['sub_pred']).astype(np.float64)
    q, _ = _queries(ctx, subject)
    allowed = _allowed(quads, q, subject, case, num_e)
    known = None if case == 'none' else quads if case == 'time_aware' else quads[:, :3]
    for k in (5, num_e):
        vals, ids = _forecast(ctx, subject, k, known, case == 'time_aware')
        assert vals.dtype == torch.float32 and ids.dtype == torch.long
        n_band = check_against_scores(vals, ids, z, allowed, k, 1e-6, 1e-5)
        assert n_band <= len(z) // 10, (k, n_band)
        if case != 'none' and k == num_e:
            assert (ids < 0).any(dim=1).all()                    # every triple's own answer is known


def test_answer_sits_at_the_raw_rank():
    ctx = _ctx()
    m, quads, rows = ctx['model'], ctx['quads'], ctx['gold']['rows']
    q = quads[rows]
    sh = synthetic.observed_history(quads, q[:, 0], q[:, 3], True)
    oh = synthetic.observed_history(quads, q[:, 2], q[:, 3], False)
    raw = m.evaluate_observed(q, sh, oh, ctx['gd'], ctx['ge'], raw=True)['ranks'].reshape(-1, 2)     # [sub, ob]
    checked = 0
    for subject, col, label in ((True, 1, q[:, 2]), (False, 0, q[:, 0])):
        vals, ids = _forecast(ctx, subject, m.in_dim)
        vals, ids = vals.numpy(), ids.numpy()
        for j in range(len(q)):
            rank = raw[j, col]
            if rank != int(rank):
                continue                                        # a tie in z
            pos = int(rank) - 1
            v = vals[j]
            if (pos > 0 and v[pos - 1] == v[pos]) or (pos + 1 < len(v) and v[pos + 1] == v[pos]):
                continue                                        # a tie in p: its order is by id
            assert ids[j, pos] == label[j], (subject, j, pos)
            checked += 1
    assert checked >= len(q), checked


def _brute_window(facts, e, t, subject, history_len):
    fix, other = (0, 2) if subject else (2, 0)
    mine = facts[facts[:, fix] == e]
    ts = np.unique(mine[mine[:, 3] < t, 3])[-history_len:]
    return [mine[mine[:, 3] == x][:, [1, other]] for x in ts], ts.tolist()


@pytest.mark.parametrize('preset,timestamps', [('tiny', None), ('icews18', 20)])
def test_observed_history_equals_build_history(preset, timestamps):
    quads, num_e, _ = synthetic.make_quads(preset, seed=5, num_timestamps=timestamps)
    for S, ST, O, OT in (synthetic.build_history(quads), restate.build_history(quads, num_e)):
        for (lists, times), (ref, ref_t) in ((synthetic.observed_history(quads, quads[:, 0], quads[:, 3], True), (S, ST)),
                                             (synthetic.observed_history(quads, quads[:, 2], quads[:, 3], False), (O, OT))):
            assert len(lists) == len(times) == len(quads)
            for i in range(len(quads)):
                assert times[i] == ref_t[i] and all(type(x) is int for x in times[i]), i
                assert len(lists[i]) == len(ref[i]), i
                for a, b in zip(lists[i], ref[i]):
                    assert a.dtype == np.int64 and a.shape == b.shape and np.array_equal(a, b), i


def test_observed_history_shares_one_array_per_entity_timestamp():
    quads, _, _ = synthetic.make_quads('tiny', seed=5)
    for subject, c in ((True, 0), (False, 2)):
        lists, times = synthetic.observed_history(quads, quads[:, c], quads[:, 3], subject)
        objs, entries = {}, 0
        for e, hl, ht in zip(quads[:, c].tolist(), lists, times):
            for a, t in zip(hl, ht):
                entries += 1
                assert objs.setdefault((e, t), a) is a, (e, t)
        assert len(objs) < entries                              # windows do share entries


def test_observed_history_sees_only_earlier_timestamps():
    """Queries in the middle of a timestamp (the facts of t itself known), between timestamps, before the first and past the
    last, against a scan of the facts; a short history_len cuts the window."""
    quads, num_e, _ = synthetic.make_quads('tiny', seed=5)
    times = np.unique(quads[:, 3])
    rng = np.random.RandomState(0)
    ts = np.concatenate((quads[rng.choice(len(quads), 60), 3], rng.choice(times, 20) + 5, [times[0] - 1, times[0],
                                                                                             times[-1] + 1]))
    ents = np.concatenate((quads[rng.choice(len(quads), 60), 0], rng.randint(0, num_e, len(ts) - 60)))
    for subject in (True, False):
        for history_len in (3, 10):
            lists, got_t = synthetic.observed_history(quads, ents, ts, subject, history_len)
            for i, (e, t) in enumerate(zip(ents, ts)):
                ref, ref_t = _brute_window(quads, e, t, subject, history_len)
                assert got_t[i] == ref_t and all(x < t for x in got_t[i]), i
                assert len(lists[i]) == len(ref) and all(np.array_equal(a, b) for a, b in zip(lists[i], ref)), i
    mid = ts[:60]
    assert np.isin(mid, times).all()                           # the first queries sit on timestamps with known facts
    with pytest.raises(ValueError, match='quadruples'):
        synthetic.observed_history(quads[:, :3], ents, ts)
    with pytest.raises(ValueError, match='timestamps'):
        synthetic.observed_history(quads, ents, ts[:-1])


def test_chunk_size_and_query_order_change_no_bit(monkeypatch):
    from renet_b200 import inference
    ctx = _ctx()
    quads = ctx['quads']
    ref = _forecast(ctx, True, 7, quads, True)
    monkeypatch.setattr(inference, 'OBSERVED_RANK_ROWS', 3)
    got = _forecast(ctx, True, 7, quads, True)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    monkeypatch.undo()
    rows = ctx['gold']['rows']
    perm = np.random.RandomState(1).permutation(len(rows))
    vals, ids = _forecast(ctx, True, 7, quads, True, rows=rows[perm])
    assert torch.equal(vals, ref[0][perm]) and torch.equal(ids, ref[1][perm])


@pytest.mark.parametrize('training', [False, True])
def test_forecast_observed_leaves_state_and_rng_unchanged(training):
    ctx = _ctx()
    m = ctx['model']
    m.latest_time = torch.tensor(ctx['t_test'])
    m.train(training)
    before = {k: copy.deepcopy(getattr(m, k)) for k in STATE}
    gd_keys, gd_vals = list(m.graph_dict.keys()), list(m.graph_dict.values())
    ge_keys, ge_vals = list(m.global_emb.keys()), [v.clone() for v in m.global_emb.values()]
    arg_gd, arg_ge = dict(ctx['gd']), {t: v.clone() for t, v in ctx['ge'].items()}
    torch.manual_seed(99)
    rng = torch.get_rng_state()
    _forecast(ctx, False, 5, ctx['quads'], True)
    assert torch.equal(torch.get_rng_state(), rng)
    assert m.training == training and all(mod.training == training for mod in m.modules())
    for k in STATE:
        assert _same(getattr(m, k), before[k]), k
    assert list(m.graph_dict.keys()) == gd_keys and all(a is b for a, b in zip(m.graph_dict.values(), gd_vals))
    assert list(m.global_emb.keys()) == ge_keys and all(torch.equal(a, b) for a, b in zip(m.global_emb.values(), ge_vals))
    assert ctx['gd'] == arg_gd and all(torch.equal(ctx['ge'][t], v) for t, v in arg_ge.items())


def test_forecast_observed_argument_errors_come_before_any_work():
    ctx = _ctx()
    m, quads = ctx['model'], ctx['quads']

    def boom(*a, **k):
        raise AssertionError('work started before the arguments were checked')
    m.aggregator.encode = boom
    m._encode_queries = boom
    m._topk_rows = boom
    q, h = _queries(ctx, True)
    n = len(q)
    k_ = next(i for i in range(n) if len(h[0][i]) >= 2)
    e, t = int(q[k_, 0]), int(h[1][k_][-1])

    def with_h(i, lists=None, times=None):
        a, b = list(h[0]), list(h[1])
        if lists is not None:
            a[i] = lists
        if times is not None:
            b[i] = times
        return (a, b)

    odd = np.asarray(h[0][k_][-1]).copy(); odd[0, 1] = (odd[0, 1] + 1) % m.in_dim
    big = np.asarray(h[0][k_][-1]).copy(); big[0, 0] = m.num_rels
    late = q.copy(); late[k_, 2] = t                                     # a history entry at the query's own timestamp
    later = q.copy(); later[k_, 2] = t - 1
    assert any(i != k_ and int(q[i, 0]) == e and t in h[1][i] for i in range(n))
    cases = [
        ((q[:, :2], h), {}, 'integer rows'),
        ((q.astype(np.float32), h), {}, 'integer rows'),
        ((q + np.array([m.in_dim, 0, 0]), h), {}, 'entity ids'),
        ((q + np.array([0, m.num_rels, 0]), h), {}, 'relation ids'),
        ((q, h), {'k': 0}, 'k = 0'),
        ((q, h), {'k': m.in_dim + 1}, 'k = %d' % (m.in_dim + 1)),
        ((q[:-1], h), {}, 'history must be'),
        ((q, (h[0][:-1], h[1])), {}, 'history must be'),
        ((q, (h[0],)), {}, 'history must be'),
        ((q, with_h(k_, times=h[1][k_][:-1])), {}, 'timestamps'),
        ((q, with_h(k_, lists=h[0][k_][:-1] + [big])), {}, 'outside'),
        ((q, with_h(k_, lists=h[0][k_][:-1] + [odd])), {}, 'differs'),
        ((late, h), {}, 'not before its query'),
        ((later, h), {}, 'not before its query'),
        ((q, h), {'graph_dict': {tt: g for tt, g in ctx['gd'].items() if tt != t}}, 'which graph_dict lacks'),
        ((q, h), {'global_emb': {tt: v for tt, v in ctx['ge'].items() if tt != t}}, 'which global_emb lacks'),
        ((q, h), {'time_aware': True}, 'time_aware needs known'),
        ((q, h), {'known': quads[:, :3], 'time_aware': True}, 'quadruples'),
        ((q, h), {'known': quads[:, :2]}, 'triples'),
    ]
    for args, kw, msg in cases:
        kw = dict(kw)
        gd, ge = kw.pop('graph_dict', ctx['gd']), kw.pop('global_emb', ctx['ge'])
        with pytest.raises(ValueError, match=msg):
            m.forecast_observed(*args, gd, ge, **kw)
