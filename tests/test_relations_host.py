"""not gpu: the relation head's calls (renet_b200/inference.py: evaluate_relations_observed, forecast_relations_observed,
forecast_relations, RelationFilterIndex) with the model on the host, the CPU oracle standing in for the CUDA encode as in
test_eval_observed_host.py and test_forecast_host.py.

* Against tests/golden/renet_relations_observed.npz (the unmodified reference's inp_r -> encoder_r -> linear_r per triple
  and direction over its own history): raw, filtered and time-aware relation ranks exact, logits and loss to 1e-5;
  forecast_relations_observed's ids exact and values to 1e-5, and the known relations left out, statically and time-aware.
* evaluate_relations_observed against a per-triple restatement (_encode_one's s_q, linear_r, rank_with_ties, filters found
  by scanning the quadruples), with repeated queries and empty histories, one encode per distinct (entity, history).
* forecast_relations against a per-query restatement over the same roll-overs; its end state and RNG equal forecast's.
* Over gloo at world size 2 every rank returns the one-process result bit for bit.
* Every documented ValueError comes before any work; the state, RNG and module mode are left as they were."""
import copy

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from helpers import load_npz, rel_err
from test_eval_batched_host import _assert_same_state, _state
from test_eval_batched_host import _ctx as _stream_ctx
from test_eval_observed_host import STATE, _ctx, _same, _split
from test_eval_sharded_host import _free_port, _stream
from test_forecast_observed_host import check_against_scores

from renet_b200 import synthetic
from renet_b200.inference import PROTOCOLS, RelationFilterIndex, rank_with_ties


def _rctx():
    ctx = _ctx()
    ctx['rgold'] = load_npz('renet_relations_observed.npz')
    return ctx


def _known_relations(quads, e, subject, t=None):
    """The relations of every known (e, r, .) (subject) or (., r, e), at t when given, by a scan of the quadruples."""
    sel = quads[:, 0 if subject else 2] == e
    if t is not None:
        sel &= quads[:, 3] == t
    return np.unique(quads[sel, 1])


def _filtered_rank(z, label, known):
    """model.py:391-405 with relations as the answers."""
    p = torch.sigmoid(torch.as_tensor(z, dtype=torch.float32))
    ground = p[label].clone()
    p[torch.as_tensor(known, dtype=torch.long)] = 0
    p[label] = ground
    return rank_with_ties(p, label)


def _allowed(quads, q, subject, case, R):
    """bool [n, R]: the relations each (entity, timestamp) query may return."""
    out = np.ones((len(q), R), dtype=bool)
    if case != 'none':
        for i, (e, t) in enumerate(q):
            out[i, _known_relations(quads, e, subject, t if case == 'time_aware' else None)] = False
    return out


# ---- evaluate_relations_observed -----------------------------------------------------------------------------------------
def test_relations_observed_matches_reference_golden():
    ctx = _rctx()
    m, gold = ctx['model'], ctx['rgold']
    rows = gold['rows']
    assert gold['s_empty'].any()                             # the golden covers empty histories
    scores = []
    lin = m.linear_r.forward
    m.linear_r.forward = lambda x: scores.append(lin(x)) or scores[-1]
    out = m.evaluate_relations_observed(*_split(ctx, rows), ctx['gd'], ctx['ge'], total_data=ctx['quads'], time_aware=True)
    m.linear_r.forward = lin
    n = len(rows)
    for key, gk in (('raw', 'raw'), ('filtered', 'filt'), ('time_filtered', 'time_filt')):
        np.testing.assert_array_equal(out['protocols'][key]['ranks'], gold[gk].reshape(-1), err_msg=key)
    np.testing.assert_array_equal(out['ranks'], gold['filt'].reshape(-1))          # raw=False: top level is filtered
    z = torch.stack(scores).detach().numpy()
    assert z.shape == (2 * n, m.num_rels)                   # one chunk: subject rows, then object rows
    assert np.abs(z[:n] - gold['z_s']).max() <= 1e-5
    assert np.abs(z[n:] - gold['z_o']).max() <= 1e-5
    assert rel_err(out['loss'], float(gold['loss'].astype(np.float64).sum())) < 1e-5
    assert set(out) >= {'mrr', 'mr', 'hits@1', 'hits@3', 'hits@10', 'loss', 'ranks', 'protocols'}
    raw = m.evaluate_relations_observed(*_split(ctx, rows), ctx['gd'], ctx['ge'], raw=True)
    np.testing.assert_array_equal(raw['ranks'], gold['raw'].reshape(-1))
    assert 'protocols' not in raw


def _with_repeats_and_empties(ctx):
    q, sh, oh = _split(ctx, ctx['rgold']['rows'])
    extra = [0, 3, 3, 17, 40]
    q = np.concatenate((q, q[extra], q[[5, 9]]))
    sh = (sh[0] + [sh[0][i] for i in extra] + [[], sh[0][9]], sh[1] + [sh[1][i] for i in extra] + [[], sh[1][9]])
    oh = (oh[0] + [oh[0][i] for i in extra] + [oh[0][5], []], oh[1] + [oh[1][i] for i in extra] + [oh[1][5], []])
    return q, sh, oh


def test_relations_observed_matches_per_triple_restatement():
    ctx = _rctx()
    m, gd, ge, quads = ctx['model'], ctx['gd'], ctx['ge'], ctx['quads']
    q, sh, oh = _with_repeats_and_empties(ctx)
    ref = {k: [] for k in PROTOCOLS}
    loss = 0.0
    with torch.no_grad():
        for i, (s, r, o, t) in enumerate(q.tolist()):
            for e, (hl, ht), subject in ((s, (sh[0][i], sh[1][i]), True), (o, (oh[0][i], oh[1][i]), False)):
                s_q = torch.zeros(m.h_dim) if len(hl) == 0 else m._encode_one(e, r, hl, ht, subject, gd, ge, relation=True)
                z = m.linear_r(torch.cat((m.ent_embeds[e], s_q)))
                loss += float(m.criterion(z.view(1, -1), torch.tensor([r])))
                ref['raw'].append(rank_with_ties(z, r))
                ref['filtered'].append(_filtered_rank(z, r, _known_relations(quads, e, subject)))
                ref['time_filtered'].append(_filtered_rank(z, r, _known_relations(quads, e, subject, t)))
    calls = []
    enc = m.aggregator.encode
    m.aggregator.encode = lambda *a, **k: calls.append(1) or enc(*a, **k)
    got = m.evaluate_relations_observed(q, sh, oh, gd, ge, total_data=quads, time_aware=True)
    m.aggregator.encode = enc
    for k in PROTOCOLS:
        np.testing.assert_array_equal(got['protocols'][k]['ranks'], np.asarray(ref[k]), err_msg=k)
    assert rel_err(got['loss'], loss) < 1e-5
    # s_q does not depend on r: one encode per distinct (entity, timestamps) of each direction
    distinct = sum(len({(int(q[i, c]), tuple(h[1][i])) for i in range(len(q)) if len(h[0][i])}) for c, h in ((0, sh), (2, oh)))
    assert len(calls) == distinct < 2 * len(q)


def test_relations_observed_chunks_give_the_same_ranks(monkeypatch):
    from renet_b200 import inference
    ctx = _rctx()
    q, sh, oh = _with_repeats_and_empties(ctx)
    args = (q, sh, oh, ctx['gd'], ctx['ge'])
    ref = ctx['model'].evaluate_relations_observed(*args, total_data=ctx['quads'], time_aware=True)
    monkeypatch.setattr(inference, 'OBSERVED_RANK_ROWS', 14)         # 7 triples per rank call
    got = ctx['model'].evaluate_relations_observed(*args, total_data=ctx['quads'], time_aware=True)
    for k in PROTOCOLS:
        np.testing.assert_array_equal(got['protocols'][k]['ranks'], ref['protocols'][k]['ranks'])
    assert got['loss'] == ref['loss']


def test_relation_filter_index_lists():
    quads, _, _ = synthetic.make_quads('tiny', seed=5)
    rng = np.random.RandomState(2)
    ents = np.concatenate((rng.randint(0, quads[:, [0, 2]].max() + 1, 40), [-1, 10 ** 6]))
    ts = np.concatenate((quads[rng.choice(len(quads), 30), 3], rng.randint(-3, quads[:, 3].max() + 5, 12)))
    for time_aware in (False, True):
        ix = RelationFilterIndex(quads if time_aware else quads[:, :3], time_aware)
        for subject in (True, False):
            b, e = ix.ranges(subject, ents, *((ts,) if time_aware else ()))
            col = ix.col(subject)
            assert col.dtype == np.int32
            for i in range(len(ents)):
                ref = _known_relations(quads, ents[i], subject, ts[i] if time_aware else None)
                np.testing.assert_array_equal(col[b[i]:e[i]], ref, err_msg=str((time_aware, subject, i)))
    with pytest.raises(ValueError, match='quadruples'):
        RelationFilterIndex(quads[:, :3], time_aware=True)


def test_relations_observed_leaves_state_and_rng_unchanged():
    ctx = _rctx()
    m = ctx['model']
    m.latest_time = torch.tensor(ctx['t_test'])
    m.train(True)
    before = {k: copy.deepcopy(getattr(m, k)) for k in STATE}
    torch.manual_seed(99)
    rng = torch.get_rng_state()
    m.evaluate_relations_observed(*_split(ctx, ctx['rgold']['rows']), ctx['gd'], ctx['ge'], total_data=ctx['quads'],
                                  time_aware=True)
    q, hist = _rqueries(ctx, False)
    m.forecast_relations_observed(q, hist, ctx['gd'], ctx['ge'], k=3, subject=False, known=ctx['quads'], time_aware=True)
    assert torch.equal(torch.get_rng_state(), rng)
    assert all(mod.training for mod in m.modules())
    for k in STATE:
        assert _same(getattr(m, k), before[k]), k


# ---- forecast_relations_observed -----------------------------------------------------------------------------------------
def _rqueries(ctx, subject, rows=None):
    """The golden's triples as (entity, timestamp) queries of one direction, with histories built from the facts."""
    quads = ctx['quads']
    q = quads[ctx['rgold']['rows'] if rows is None else rows]
    c = 0 if subject else 2
    return np.stack((q[:, c], q[:, 3]), 1), synthetic.observed_history(quads, q[:, c], q[:, 3], subject)


@pytest.mark.parametrize('case', ['none', 'static', 'time_aware'])
@pytest.mark.parametrize('subject', [True, False])
def test_forecast_relations_observed_matches_reference_golden(subject, case):
    ctx = _rctx()
    m, quads, gold = ctx['model'], ctx['quads'], ctx['rgold']
    R = m.num_rels
    q, hist = _rqueries(ctx, subject)
    side = 's' if subject else 'o'
    known = None if case == 'none' else quads if case == 'time_aware' else quads[:, :3]
    vals, ids = m.forecast_relations_observed(q, hist, ctx['gd'], ctx['ge'], k=R, subject=subject, known=known,
                                              time_aware=case == 'time_aware')
    assert vals.dtype == torch.float32 and ids.dtype == torch.long and vals.shape == (len(q), R)
    if case == 'none':
        np.testing.assert_array_equal(ids.numpy(), gold['topk_ids_' + side])
        assert np.abs(vals.numpy() - gold['topk_vals_' + side]).max() <= 1e-5
    z = gold['z_' + side].astype(np.float64)
    allowed = _allowed(quads, q, subject, case, R)
    for k in (1, 3, R):
        v, i = m.forecast_relations_observed(q, hist, ctx['gd'], ctx['ge'], k=k, subject=subject, known=known,
                                             time_aware=case == 'time_aware')
        assert check_against_scores(v, i, z, allowed, k, 1e-6, 1e-5) == 0
    if case != 'none':
        assert (ids < 0).any(dim=1).all()                       # every triple's own relation is known


def test_forecast_relations_observed_argument_errors_come_before_any_work():
    ctx = _rctx()
    m, quads = ctx['model'], ctx['quads']

    def boom(*a, **k):
        raise AssertionError('work started before the arguments were checked')
    m.aggregator.encode = boom
    m._encode_queries = boom
    m._topk_rows = boom
    m._rank_rows = boom
    q, h = _rqueries(ctx, True)
    n = len(q)
    k_ = next(i for i in range(n) if len(h[0][i]) >= 2)
    t = int(h[1][k_][-1])
    big = np.asarray(h[0][k_][-1]).copy(); big[0, 0] = m.num_rels
    late = q.copy(); late[k_, 1] = t
    cases = [
        ((q[:, :1], h), {}, 'integer rows'),
        ((np.concatenate((q, q[:, :1]), 1), h), {}, 'integer rows'),
        ((q.astype(np.float32), h), {}, 'integer rows'),
        ((q + np.array([m.in_dim, 0]), h), {}, 'entity ids'),
        ((q, h), {'k': 0}, 'k = 0'),
        ((q, h), {'k': m.num_rels + 1}, 'k = %d' % (m.num_rels + 1)),
        ((q[:-1], h), {}, 'history must be'),
        ((q, (h[0],)), {}, 'history must be'),
        ((q, (h[0], h[1][:k_] + [h[1][k_][:-1]] + h[1][k_ + 1:])), {}, 'timestamps'),
        ((q, (h[0][:k_] + [h[0][k_][:-1] + [big]] + h[0][k_ + 1:], h[1])), {}, 'outside'),
        ((late, h), {}, 'not before its query'),
        ((q, h), {'graph_dict': {tt: g for tt, g in ctx['gd'].items() if tt != t}}, 'which graph_dict lacks'),
        ((q, h), {'global_emb': {tt: v for tt, v in ctx['ge'].items() if tt != t}}, 'which global_emb lacks'),
        ((q, h), {'time_aware': True}, 'time_aware needs known'),
        ((q, h), {'known': quads[:, :3], 'time_aware': True}, 'quadruples'),
        ((q, h), {'known': quads[:, :2]}, 'triples'),
    ]
    for args, kw, msg in cases:
        kw = dict(dict(k=3), **kw)                               # the default k = 10 is above the tiny model's 6 relations
        gd, ge = kw.pop('graph_dict', ctx['gd']), kw.pop('global_emb', ctx['ge'])
        with pytest.raises(ValueError, match=msg) as err:
            m.forecast_relations_observed(*args, gd, ge, **kw)
        assert str(err.value).startswith('forecast_relations_observed: '), str(err.value)
    # evaluate_relations_observed: evaluate_observed's checks, named for the call
    S, ST, O, OT = ctx['hist']
    rows = ctx['rgold']['rows']
    sh, oh = ([S[i] for i in rows], [ST[i] for i in rows]), ([O[i] for i in rows], [OT[i] for i in rows])
    tq = quads[rows]
    ecases = [
        ((tq[:, :3], sh, oh), {}, 'quadruples'),
        ((tq, sh, oh), {}, 'needs total_data'),
        ((tq, sh, oh), {'time_aware': True, 'total_data': quads[:, :3]}, 'time column'),
        ((tq, (sh[0][:-1], sh[1]), oh), {'raw': True}, 's_history must be'),
        ((tq + np.array([0, 0, m.in_dim, 0]), sh, oh), {'raw': True}, 'entity ids'),
        ((tq + np.array([0, m.num_rels, 0, 0]), sh, oh), {'raw': True}, 'relation ids'),
        ((tq, sh, oh), {'raw': True, 'graph_dict': {}}, 'which graph_dict lacks'),
    ]
    for args, kw, msg in ecases:
        kw = dict(kw)
        gd, ge = kw.pop('graph_dict', ctx['gd']), kw.pop('global_emb', ctx['ge'])
        with pytest.raises(ValueError, match=msg):
            m.evaluate_relations_observed(*args, gd, ge, **kw)


# ---- forecast_relations over the test-time state -------------------------------------------------------------------------
CASES = {'none': dict(), 'static': dict(known=True), 'time_aware': dict(known=True, time_aware=True)}


def _squeries(ctx, subject, te=None):
    quads = ctx['quads']
    te = _stream(ctx) if te is None else te
    q = quads[te]
    return np.stack((q[:, 0] if subject else q[:, 2], q[:, 3]), 1)


def _forecast_relations(ctx, subject, case, k, group=None, seed=1234):
    m, quads = ctx['model'], ctx['quads']
    q = _squeries(ctx, subject)
    m.latest_time = torch.tensor(int(q[0, 1]))
    torch.manual_seed(seed)
    kw = dict(CASES[case])
    if kw.pop('known', False):
        kw['known'] = quads
    return m.forecast_relations(q, ctx['gm'], k=k, subject=subject, process_group=group, **kw)


def _restated_relations(ctx, subject, case, k):
    m, quads, gm = ctx['model'], ctx['quads'], ctx['gm']
    q = _squeries(ctx, subject)
    m.latest_time = torch.tensor(int(q[0, 1]))
    torch.manual_seed(1234)
    m._trim_test_histories()
    vals, ids = [], []
    with torch.no_grad():
        for e, t in q:
            if int(m.latest_time) != int(t):
                m._roll_over(torch.tensor(int(t)), gm)
            hist, hist_t = (m.s_hist_test, m.s_hist_test_t) if subject else (m.o_hist_test, m.o_hist_test_t)
            s_q = (torch.zeros(m.h_dim) if len(hist[e]) == 0
                   else m._encode_one(int(e), 0, hist[e], hist_t[e], subject, relation=True))
            p = torch.softmax(m.linear_r(torch.cat((m.ent_embeds[int(e)], s_q))).view(1, -1), dim=1).view(-1).numpy()
            cols = np.arange(len(p))
            if case != 'none':
                cols = np.setdiff1d(cols, _known_relations(quads, e, subject, t if case == 'time_aware' else None))
            order = cols[np.lexsort((cols, -p[cols]))][:k]
            v = np.zeros(k, np.float32)
            i = np.full(k, -1, np.int64)
            v[:len(order)], i[:len(order)] = p[order], order
            vals.append(v)
            ids.append(i)
    return np.stack(vals), np.stack(ids)


@pytest.mark.parametrize('case', list(CASES))
@pytest.mark.parametrize('subject', [True, False])
def test_forecast_relations_equals_per_query_restatement(subject, case):
    R = _stream_ctx()['model'].num_rels
    for k in (3, R):
        a, b = _stream_ctx(), _stream_ctx()
        v, i = _forecast_relations(a, subject, case, k)
        rv, ri = _restated_relations(b, subject, case, k)
        assert v.dtype == torch.float32 and i.dtype == torch.long and v.shape == (len(rv), k)
        np.testing.assert_array_equal(i.numpy(), ri)
        np.testing.assert_array_equal(v.numpy(), rv)
        _assert_same_state(_state(a), _state(b))
    if case != 'none':
        assert (i < 0).any(dim=1).all()                          # k = R: each entity's own relation is known


def test_state_after_forecast_relations_equals_forecast():
    """The same roll-overs: forecast_relations leaves the state and RNG stream forecast leaves over the same timestamps."""
    a, b = _stream_ctx(), _stream_ctx()
    _forecast_relations(a, True, 'static', 4)
    m, quads = b['model'], b['quads']
    te = _stream(b)
    q = np.stack((quads[te, 0], quads[te, 1], quads[te, 3]), 1)
    m.latest_time = torch.tensor(int(q[0, 2]))
    torch.manual_seed(1234)
    m.forecast(q, b['gm'], k=4, known=quads)
    assert len(np.unique(quads[te, 3])) == 3                 # two roll-overs
    _assert_same_state(_state(a), _state(b))


def test_forecast_relations_bad_queries_raise():
    ctx = _stream_ctx()
    m = ctx['model']
    q = _squeries(ctx, True)
    m.latest_time = torch.tensor(int(q[0, 1]))
    bad = {'rows': q[:, :1], 'three': np.concatenate((q, q[:, :1]), 1), 'float': q.astype(np.float32),
           'entity': q + np.array([m.in_dim, 0]), 'order': q[::-1], 'past': q - np.array([0, 1])}
    for name, qq in bad.items():
        with pytest.raises(ValueError, match='forecast_relations'):
            m.forecast_relations(np.ascontiguousarray(qq), ctx['gm'], k=3)
    for k in (0, m.num_rels + 1):
        with pytest.raises(ValueError, match='k = '):
            m.forecast_relations(q, ctx['gm'], k=k)
    with pytest.raises(ValueError, match='time_aware'):
        m.forecast_relations(q, ctx['gm'], k=3, time_aware=True)
    assert int(m.latest_time) == int(q[0, 1])                # nothing ran


def _sharded_worker(rank, port, world, out):
    import os
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        for subject in (True, False):
            for case in CASES:
                ctx = _stream_ctx()
                v, i = _forecast_relations(ctx, subject, case, 4, group=dist.group.WORLD)
                out[(subject, case, rank)] = (v, i, _state(ctx))
    finally:
        dist.destroy_process_group()


def test_sharded_forecast_relations_equals_single_process():
    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_sharded_worker, args=(_free_port(), world, out), nprocs=world, join=True)
    res = dict(out)
    mgr.shutdown()
    for subject in (True, False):
        for case in CASES:
            ctx = _stream_ctx()
            v, i = _forecast_relations(ctx, subject, case, 4)
            ref_state = _state(ctx)
            for rank in range(world):
                gv, gi, state = res[(subject, case, rank)]
                assert gv.dtype == v.dtype and gi.dtype == i.dtype
                assert torch.equal(gv, v) and torch.equal(gi, i), (subject, case, rank)
                _assert_same_state(state, ref_state)
