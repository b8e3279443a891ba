"""not gpu: RENet.evaluate_observed (renet_b200/inference.py) with the model on the host, the CPU oracle standing in for the
CUDA encode as in test_inference_host.py.

* Against tests/golden/renet_eval_observed.npz (the unmodified reference's RGCNAggregator.predict + encoder + linear per
  triple over its own ground-truth history): raw, filtered and time-aware ranks exact, scores to 1e-5.
* Against a per-triple restatement built from _encode_one and rank_with_ties, with empty histories and repeated queries.
* The test-time state, torch's RNG and the module's mode are unchanged by the call.
* Every argument error is a ValueError raised before any encoding or ranking.
* The device batcher's plan for a split holds one component per distinct (entity, history timestamp)."""
import copy

import numpy as np
import pytest
import torch

from helpers import eval_setup, load_npz, rel_err
from test_inference_host import _oracle_encode

from renet_b200 import synthetic
from renet_b200.inference import PROTOCOLS, _chunk_view, _same_time, rank_with_ties


def _ctx():
    ctx = eval_setup('cpu')
    ctx['model'].aggregator.encode = _oracle_encode(ctx)
    ctx['gold'] = load_npz('renet_eval_observed.npz')
    quads = ctx['quads']
    ctx['gd'] = synthetic.build_graph_dict(quads, ctx['dims'][1])          # the true graphs of every timestamp
    ctx['ge'] = dict(ctx['model'].global_emb)
    return ctx


def _split(ctx, rows):
    S, ST, O, OT = ctx['hist']
    return (ctx['quads'][rows], ([S[i] for i in rows], [ST[i] for i in rows]), ([O[i] for i in rows], [OT[i] for i in rows]))


def _observed(ctx, q, sh, oh, **kw):
    return ctx['model'].evaluate_observed(q, sh, oh, ctx['gd'], ctx['ge'], **kw)


def test_observed_matches_reference_golden():
    ctx = _ctx()
    m, gold = ctx['model'], ctx['gold']
    rows = gold['rows']
    assert gold['s_empty'].any()                             # the golden covers empty histories
    scores = []
    lin = m.linear.forward
    m.linear.forward = lambda x: scores.append(lin(x)) or scores[-1]
    out = _observed(ctx, *_split(ctx, rows), total_data=ctx['quads'], time_aware=True)
    m.linear.forward = lin
    n = len(rows)
    for key, gk in (('raw', 'raw'), ('filtered', 'filt'), ('time_filtered', 'time_filt')):
        np.testing.assert_array_equal(out['protocols'][key]['ranks'], gold[gk].reshape(-1), err_msg=key)
    np.testing.assert_array_equal(out['ranks'], gold['filt'].reshape(-1))          # raw=False: top level is filtered
    z = torch.stack(scores).detach().numpy()
    assert z.shape[0] == 2 * n                              # one chunk: object rows, then subject rows
    assert np.abs(z[:n] - gold['ob_pred']).max() <= 1e-5
    assert np.abs(z[n:] - gold['sub_pred']).max() <= 1e-5
    assert rel_err(out['loss'], float(gold['loss'].astype(np.float64).sum())) < 1e-5
    raw = _observed(ctx, *_split(ctx, rows), raw=True)
    np.testing.assert_array_equal(raw['ranks'], gold['raw'].reshape(-1))


def _restated(ctx, q, sh, oh, known):
    """Per triple: _encode_one over the triple's own histories (zero when empty), ``linear`` in both directions, then
    rank_with_ties raw and _filtered_ranks against ``known`` and against its rows at the triple's timestamp."""
    m, gd, ge = ctx['model'], ctx['gd'], ctx['ge']
    R, h = m.num_rels, m.h_dim
    out = {k: [] for k in PROTOCOLS}
    loss = 0.0
    with torch.no_grad():
        for i, trip in enumerate(torch.from_numpy(q)):
            s, r, o = (int(x) for x in trip[:3])
            s_h = torch.zeros(h) if len(sh[0][i]) == 0 else m._encode_one(s, r, sh[0][i], sh[1][i], True, gd, ge)
            o_h = torch.zeros(h) if len(oh[0][i]) == 0 else m._encode_one(o, r, oh[0][i], oh[1][i], False, gd, ge)
            ob = m.linear(torch.cat((m.ent_embeds[s], s_h, m.rel_embeds[:R][r])))
            sub = m.linear(torch.cat((m.ent_embeds[o], o_h, m.rel_embeds[R:][r])))
            loss += float(m.criterion(ob.view(1, -1), torch.tensor([o])) + m.criterion(sub.view(1, -1), torch.tensor([s])))
            out['raw'].append([rank_with_ties(sub, s), rank_with_ties(ob, o)])
            out['filtered'].append(m._filtered_ranks(trip, sub, ob, known))
            out['time_filtered'].append(m._filtered_ranks(trip, sub, ob, _same_time(known, trip)))
    return {k: np.concatenate([np.asarray(x, dtype=np.float64) for x in v]) for k, v in out.items()}, loss


def _with_repeats_and_empties(ctx):
    """The golden's rows, then five of them again (repeated queries), then two with their histories emptied."""
    q, sh, oh = _split(ctx, ctx['gold']['rows'])
    extra = [0, 3, 3, 17, 40]
    q = np.concatenate((q, q[extra], q[[5, 9]]))
    sh = (sh[0] + [sh[0][i] for i in extra] + [[], sh[0][9]], sh[1] + [sh[1][i] for i in extra] + [[], sh[1][9]])
    oh = (oh[0] + [oh[0][i] for i in extra] + [oh[0][5], []], oh[1] + [oh[1][i] for i in extra] + [oh[1][5], []])
    return q, sh, oh


def test_observed_matches_per_triple_restatement():
    ctx = _ctx()
    m = ctx['model']
    q, sh, oh = _with_repeats_and_empties(ctx)
    ref, ref_loss = _restated(ctx, q, sh, oh, torch.from_numpy(ctx['quads']))
    calls = []
    enc = m.aggregator.encode
    m.aggregator.encode = lambda *a, **k: calls.append(1) or enc(*a, **k)
    got = _observed(ctx, q, sh, oh, total_data=ctx['quads'], time_aware=True)
    m.aggregator.encode = enc
    for k in PROTOCOLS:
        np.testing.assert_array_equal(got['protocols'][k]['ranks'], ref[k], err_msg=k)
    assert rel_err(got['loss'], ref_loss) < 1e-5
    # equal queries are encoded once: one call per distinct (entity, relation, timestamps) of each direction
    distinct = sum(len({(int(q[i, c]), int(q[i, 1]), tuple(h[1][i])) for i in range(len(q)) if len(h[0][i])})
                   for c, h in ((0, sh), (2, oh)))
    assert len(calls) == distinct < 2 * len(q)


def test_observed_chunks_give_the_same_ranks(monkeypatch):
    from renet_b200 import inference
    ctx = _ctx()
    q, sh, oh = _with_repeats_and_empties(ctx)
    ref = _observed(ctx, q, sh, oh, total_data=ctx['quads'], time_aware=True)
    monkeypatch.setattr(inference, 'OBSERVED_RANK_ROWS', 14)         # 7 triples per rank call
    got = _observed(ctx, q, sh, oh, total_data=ctx['quads'], time_aware=True)
    for k in PROTOCOLS:
        np.testing.assert_array_equal(got['protocols'][k]['ranks'], ref['protocols'][k]['ranks'], err_msg=k)
    assert rel_err(got['loss'], ref['loss']) < 1e-6


STATE = ('s_hist_test', 's_hist_test_t', 'o_hist_test', 'o_hist_test_t', 's_his_cache', 'o_his_cache', 's_his_cache_t',
         'o_his_cache_t', 'latest_time')


def _same(a, b):
    if isinstance(a, (list, tuple)):
        return type(a) is type(b) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and a.dtype == b.dtype and torch.equal(a, b)
    if isinstance(a, np.ndarray):
        return isinstance(b, np.ndarray) and a.dtype == b.dtype and np.array_equal(a, b)
    return a == b


@pytest.mark.parametrize('training', [False, True])
def test_observed_leaves_state_and_rng_unchanged(training):
    ctx = _ctx()
    m = ctx['model']
    m.latest_time = torch.tensor(ctx['t_test'])
    m.train(training)
    before = {k: copy.deepcopy(getattr(m, k)) for k in STATE}
    gd_keys, gd_vals = list(m.graph_dict.keys()), list(m.graph_dict.values())
    ge_keys, ge_vals = list(m.global_emb.keys()), [v.clone() for v in m.global_emb.values()]
    torch.manual_seed(99)
    rng = torch.get_rng_state()
    _observed(ctx, *_split(ctx, ctx['gold']['rows']), total_data=ctx['quads'], time_aware=True)
    assert torch.equal(torch.get_rng_state(), rng)
    assert m.training == training and all(mod.training == training for mod in m.modules())
    for k in STATE:
        assert _same(getattr(m, k), before[k]), k
    assert list(m.graph_dict.keys()) == gd_keys and all(a is b for a, b in zip(m.graph_dict.values(), gd_vals))
    assert list(m.global_emb.keys()) == ge_keys and all(torch.equal(a, b) for a, b in zip(m.global_emb.values(), ge_vals))


def test_observed_argument_errors_come_before_any_work():
    ctx = _ctx()
    m = ctx['model']

    def boom(*a, **k):
        raise AssertionError('work started before the arguments were checked')
    m.aggregator.encode = boom
    m._rank_rows = boom
    q, sh, oh = _split(ctx, ctx['gold']['rows'])
    n = len(q)
    k = next(i for i in range(n) if len(sh[0][i]) >= 2)
    e, t = int(q[k, 0]), int(sh[1][k][-1])

    def with_s(i, lists=None, times=None):
        a, b = list(sh[0]), list(sh[1])
        if lists is not None:
            a[i] = lists
        if times is not None:
            b[i] = times
        return (a, b)

    bad_q = q.copy(); bad_q[0, 2] = m.in_dim
    bad_r = q.copy(); bad_r[1, 1] = m.num_rels
    odd = np.asarray(sh[0][k][-1]).copy(); odd[0, 1] = (odd[0, 1] + 1) % m.in_dim
    big = np.asarray(sh[0][k][-1]).copy(); big[0, 0] = m.num_rels
    gd_missing = {tt: g for tt, g in ctx['gd'].items() if tt != t}
    ge_missing = {tt: v for tt, v in ctx['ge'].items() if tt != t}
    other = next(i for i in range(n) if i != k and int(q[i, 0]) == e and t in sh[1][i]) if any(
        i != k and int(q[i, 0]) == e and t in sh[1][i] for i in range(n)) else None
    cases = [
        ((q[:-1], sh, oh), {}, 'test triples'),
        ((q, (sh[0][:-1], sh[1]), oh), {}, 's_history'),
        ((q, sh, (oh[0], oh[1][:-1])), {}, 'o_history'),
        ((q, with_s(k, times=sh[1][k][:-1]), oh), {}, 'timestamps'),
        ((bad_q, sh, oh), {}, 'entity ids'),
        ((bad_r, sh, oh), {}, 'relation ids'),
        ((q, with_s(k, lists=sh[0][k][:-1] + [big]), oh), {}, 'outside'),
        ((q, sh, oh), {'graph_dict': gd_missing}, 'timestamp %d, which graph_dict lacks' % t),
        ((q, sh, oh), {'global_emb': ge_missing}, 'timestamp %d, which global_emb lacks' % t),
        ((q, sh, oh), {'total_data': ctx['quads'][:, :3], 'time_aware': True}, 'time column'),
        ((q, sh, oh), {'total_data': None}, 'total_data'),
    ]
    if other is not None:
        # the entry of (e, t) differs between two histories that hold it
        cases.append(((q, with_s(k, lists=sh[0][k][:-1] + [odd]), oh), {}, 'differs'))
    for args, kw, msg in cases:
        kw = dict(kw)
        gd, ge = kw.pop('graph_dict', ctx['gd']), kw.pop('global_emb', ctx['ge'])
        kw.setdefault('total_data', ctx['quads'])
        with pytest.raises(ValueError, match=msg):
            m.evaluate_observed(*args, gd, ge, **kw)
    assert other is not None, 'the split should hold one (entity, timestamp) entry in two histories'


def test_plan_has_one_component_per_entity_timestamp():
    from renet_b200 import hoststore
    ctx = _ctx()
    m = ctx['model']
    q, sh, oh = _split(ctx, ctx['gold']['rows'])
    for c, (lists, times), name in ((0, sh, 's_history'), (2, oh, 'o_history')):
        (hist, hist_t, hid, ent_of), has = m._observed_histories(q[:, c], (lists, times), name, ctx['gd'], ctx['ge'])
        q_h = np.unique(hid[has])
        view, _ = _chunk_view(hist, hist_t, q_h, ent_of[q_h], ctx['gd'])
        pairs = {(int(ent_of[x]), int(t)) for x in q_h for t in hist_t[x]}
        entries = sum(len(hist_t[x]) for x in q_h)
        assert len(pairs) < entries                            # some (entity, timestamp) sits in several windows
        buf = np.zeros(1 << 20, dtype=np.int32)
        r = hoststore.plan_view_raw(view, buf)
        assert r['G'] == len(pairs), (name, r['G'], len(pairs))
        assert r['Q'] == len(q_h)
