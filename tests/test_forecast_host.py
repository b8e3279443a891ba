"""-m "not gpu": host logic of RENet.forecast (renet_b200/inference.py) on the golden stream of renet_eval_tiny.npz, with the
CPU oracle standing in for the CUDA encode as in test_eval_batched_host.py.

* forecast equals a per-query restatement -- the same roll-overs, then _encode_one, ``linear``, softmax and a stable
  descending sort with the known answers (found by scanning the triples) taken out -- in both directions, without a
  filter, with the static and the time-aware one, and with k above the admissible count (padded with -1 / 0);
* after forecast the model is in the state evaluate_stream_batched leaves over the same timestamps (RNG included);
* over gloo at world sizes 2 and 3 every rank returns the one-process result bit for bit; mismatched arguments raise."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_eval_batched_host import _assert_same_state, _ctx, _state
from test_eval_sharded_host import _free_port, _stream

CASES = {'none': dict(), 'static': dict(known=True), 'time_aware': dict(known=True, time_aware=True)}


def _queries(ctx, subject, te=None):
    """(entity, relation, timestamp) rows of the stream: the subject of each triple asks for objects, the object for
    subjects."""
    quads = ctx['quads']
    te = _stream(ctx) if te is None else te
    q = quads[te]
    return np.stack((q[:, 0] if subject else q[:, 2], q[:, 1], q[:, 3]), 1), te


def _forecast(ctx, subject, case, k, te=None, group=None, seed=1234):
    m, quads = ctx['model'], ctx['quads']
    q, te = _queries(ctx, subject, te)
    m.latest_time = torch.tensor(int(q[0, 2]))
    torch.manual_seed(seed)
    kw = dict(CASES[case])
    if kw.pop('known', False):
        kw['known'] = quads
    return m.forecast(q, ctx['gm'], k=k, subject=subject, process_group=group, **kw)


def _restated(ctx, subject, case, k):
    """The per-query restatement of forecast."""
    m, quads, gm = ctx['model'], ctx['quads'], ctx['gm']
    q, _ = _queries(ctx, subject)
    m.latest_time = torch.tensor(int(q[0, 2]))
    torch.manual_seed(1234)
    m._trim_test_histories()
    R = m.num_rels
    rel = m.rel_embeds[:R] if subject else m.rel_embeds[R:]
    vals, ids = [], []
    with torch.no_grad():
        for e, r, t in q:
            if int(m.latest_time) != int(t):
                m._roll_over(torch.tensor(int(t)), gm)
            hist, hist_t = (m.s_hist_test, m.s_hist_test_t) if subject else (m.o_hist_test, m.o_hist_test_t)
            s_h = torch.zeros(m.h_dim) if len(hist[e]) == 0 else m._encode_one(int(e), int(r), hist[e], hist_t[e], subject)
            z = m.linear(torch.cat((m.ent_embeds[int(e)], s_h, rel[int(r)])))
            p = torch.softmax(z.view(1, -1), dim=1).view(-1).numpy()
            fix, ans = (0, 2) if subject else (2, 0)
            sel = (quads[:, fix] == e) & (quads[:, 1] == r)
            if case == 'time_aware':
                sel &= quads[:, 3] == t
            cols = np.arange(len(p))
            if case != 'none':
                cols = np.setdiff1d(cols, quads[sel, ans])
            order = cols[np.lexsort((cols, -p[cols]))][:k]            # p descending, then the lower id
            v = np.zeros(k, np.float32)
            i = np.full(k, -1, np.int64)
            v[:len(order)], i[:len(order)] = p[order], order
            vals.append(v)
            ids.append(i)
    return np.stack(vals), np.stack(ids)


@pytest.mark.parametrize('case', list(CASES))
@pytest.mark.parametrize('subject', [True, False])
def test_forecast_equals_per_query_restatement(subject, case):
    a, b = _ctx(), _ctx()
    v, i = _forecast(a, subject, case, 5)
    rv, ri = _restated(b, subject, case, 5)
    assert v.dtype == torch.float32 and i.dtype == torch.long and v.shape == (len(rv), 5)
    np.testing.assert_array_equal(i.numpy(), ri)
    np.testing.assert_array_equal(v.numpy(), rv)
    assert (i >= 0).all()
    _assert_same_state(_state(a), _state(b))


@pytest.mark.parametrize('case', ['static', 'time_aware'])
def test_k_above_the_admissible_count_pads(case):
    """k = every entity: the rows with known answers have fewer admissible ones, and their last slots are -1 / 0."""
    a, b = _ctx(), _ctx()
    k = a['model'].in_dim
    v, i = _forecast(a, True, case, k)
    rv, ri = _restated(b, True, case, k)
    np.testing.assert_array_equal(i.numpy(), ri)
    np.testing.assert_array_equal(v.numpy(), rv)
    pad = i < 0
    assert pad.any(dim=1).all()                          # every query knows its own answer at least
    assert (v[pad] == 0).all()
    for row_i, row_p in zip(i, pad):                     # the padding is a suffix
        assert not row_p[:int((~row_p).sum())].any()


def test_state_after_forecast_equals_evaluation():
    a, b = _ctx(rebinding=False), _ctx(rebinding=False)
    _forecast(a, True, 'static', 10)
    m, quads = b['model'], b['quads']
    S, ST, O, OT = b['hist']
    te = _stream(b)
    m.latest_time = torch.tensor(int(quads[te[0], 3]))
    torch.manual_seed(1234)
    m.evaluate_stream_batched(quads[te], ([S[i] for i in te], [ST[i] for i in te]), ([O[i] for i in te], [OT[i] for i in te]),
                              b['gm'], total_data=quads)
    assert len(np.unique(quads[te, 3])) == 3                 # two roll-overs
    _assert_same_state(_state(a), _state(b))


def test_bad_queries_raise():
    ctx = _ctx()
    m = ctx['model']
    q, _ = _queries(ctx, True)
    m.latest_time = torch.tensor(int(q[0, 2]))
    bad = {'rows': q[:, :2], 'float': q.astype(np.float32), 'entity': q + np.array([m.in_dim, 0, 0]),
           'relation': q + np.array([0, m.num_rels, 0]), 'order': q[::-1], 'past': q - np.array([0, 0, 1])}
    for name, qq in bad.items():
        with pytest.raises(ValueError):
            m.forecast(np.ascontiguousarray(qq), ctx['gm'])
    for k in (0, m.in_dim + 1):
        with pytest.raises(ValueError, match='k = '):
            m.forecast(q, ctx['gm'], k=k)
    with pytest.raises(ValueError, match='time_aware'):
        m.forecast(q, ctx['gm'], time_aware=True)
    assert int(m.latest_time) == int(q[0, 2])                # nothing ran


# ---- sharded over gloo ---------------------------------------------------------------------------------------------------
def _init(rank, port, world):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)


def _one_query_stream(ctx):
    """A timestamp of ONE query, then the test split after a roll-over."""
    quads, ev = ctx['quads'], ctx['ev']
    va_last = ev['va'][quads[ev['va'], 3] == quads[ev['va'], 3].max()]
    return np.concatenate((va_last[:1], ev['te']))


def _sharded_worker(rank, port, world, out):
    _init(rank, port, world)
    try:
        for subject in (True, False):
            for case in CASES:
                ctx = _ctx()
                te = _one_query_stream(ctx) if world == 3 else None
                v, i = _forecast(ctx, subject, case, 7, te=te, group=dist.group.WORLD)
                out[(subject, case, rank)] = (v, i, _state(ctx))
        if world == 2:
            ctx = _ctx()
            res = {}
            for name, kw in (('k', dict(k=7 + rank)), ('subject', dict(subject=bool(rank))),
                             ('queries', dict(te=_stream(ctx)[:-1] if rank else None))):
                kw = dict(dict(subject=True, k=7, te=None), **kw)
                try:
                    _forecast(_ctx(), kw['subject'], 'static', kw['k'], te=kw['te'], group=dist.group.WORLD)
                    res[name] = None
                except ValueError as e:
                    res[name] = str(e)
            out[('mismatch', rank)] = res
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 3])
def test_sharded_forecast_equals_single_process(world):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_sharded_worker, args=(_free_port(), world, out), nprocs=world, join=True)
    res = dict(out)
    mgr.shutdown()
    for subject in (True, False):
        for case in CASES:
            ctx = _ctx()
            te = _one_query_stream(ctx) if world == 3 else None
            if world == 3:
                assert np.sum(ctx['quads'][te, 3] == ctx['quads'][te[0], 3]) == 1      # fewer rows than ranks
            v, i = _forecast(ctx, subject, case, 7, te=te)
            ref_state = _state(ctx)
            for rank in range(world):
                gv, gi, state = res[(subject, case, rank)]
                assert gv.dtype == v.dtype and gi.dtype == i.dtype
                assert torch.equal(gv, v) and torch.equal(gi, i), (subject, case, rank)
                _assert_same_state(state, ref_state)
    if world == 2:
        for rank in range(world):
            for name, msg in res[('mismatch', rank)].items():
                assert msg is not None and 'different queries' in msg, (name, rank, msg)
