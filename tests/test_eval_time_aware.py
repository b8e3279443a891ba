"""not gpu: the time-aware filter (evaluate_stream(time_aware=True), renet_b200/inference.py) -- the TimeFilterIndex against
brute-force masks, an oracle anchored on the reference's own scores, the host flow against that oracle and against the
per-triple path, the counting epilogue's SASS, and renet_decoder_rank_multi's argument checks."""
import re
import threading

import numpy as np
import pytest
import torch

from helpers import load_npz, rel_err
from test_deterministic_sass import FLOAT_ATOMIC, _matching, sass  # noqa: F401  (sass is a fixture)
from test_eval_batched_host import _assert_same_state, _ctx, _state


# ---- the index ------------------------------------------------------------------------------------------------------------
def test_time_filter_index_matches_masks():
    from renet_b200.inference import TimeFilterIndex
    rng = np.random.RandomState(7)
    times = np.asarray([0, 24, 48, 1000, 1024])
    q = np.stack((rng.randint(0, 30, 900), rng.randint(0, 6, 900), rng.randint(0, 30, 900), rng.choice(times, 900)), 1)
    q = np.concatenate((q, q[:150]))                                           # duplicates
    fi = TimeFilterIndex(q)
    n = 400
    # absent entities (30, 31), absent and out-of-range relations (-1, 6, 7), absent timestamps (-24, 12, 2000)
    probe = np.stack((rng.randint(-1, 32, n), rng.randint(-1, 8, n), rng.randint(-1, 32, n),
                      rng.choice(np.concatenate((times, [-24, 12, 2000])), n)), 1)
    probe[:50] = q[rng.randint(0, len(q), 50)]                                 # keys that are present
    for direction, col_fix, col_out in (('objects', 0, 2), ('subjects', 2, 0)):
        b, e = fi.ranges(direction, probe[:, col_fix], probe[:, 1], probe[:, 3])
        col = fi.col(direction)
        assert col.dtype == np.int32
        nonempty = 0
        for i, (s, r, o, t) in enumerate(probe):
            f = (s, r, o)[col_fix]
            known = q[(q[:, col_fix] == f) & (q[:, 1] == r) & (q[:, 3] == t)][:, col_out]
            np.testing.assert_array_equal(col[b[i]:e[i]], np.unique(known))
            nonempty += len(known) > 0
        assert nonempty >= 50
    # broadcasting of one timestamp over many keys, and an empty index
    b1, e1 = fi.ranges('objects', probe[:, 0], probe[:, 1], 48)
    b2, e2 = fi.ranges('objects', probe[:, 0], probe[:, 1], np.full(n, 48))
    assert np.array_equal(b1, b2) and np.array_equal(e1, e2)
    empty = TimeFilterIndex(np.zeros((0, 4), np.int64))
    b, e = empty.ranges('subjects', [0, 3], [0, 1], [0, 5])
    assert np.array_equal(b, e)


def test_time_filter_index_keys_do_not_overflow():
    """1 M entities x 500 relations x a GDELT-sized number of timestamps: keys stay exact."""
    from renet_b200.inference import TimeFilterIndex
    rng = np.random.RandomState(1)
    n, E, R = 20000, 1_000_000, 500
    times = np.arange(45000, dtype=np.int64) * 15                                 # 15-minute steps
    q = np.stack((rng.randint(0, E, n), rng.randint(0, R, n), rng.randint(0, E, n), rng.choice(times, n)), 1)
    q[:4, 0], q[:4, 1], q[:4, 3] = E - 1, R - 1, times[-1]                         # the largest keys
    q[:4, 2] = [5, 7, 7, 9]
    fi = TimeFilterIndex(q)
    assert fi.E * fi.R * fi.T > 1 << 40
    b, e = fi.ranges('objects', [E - 1], [R - 1], [times[-1]])
    np.testing.assert_array_equal(fi.col('objects')[b[0]:e[0]], [5, 7, 9])
    b, e = fi.ranges('objects', q[4:200, 0], q[4:200, 1], q[4:200, 3])
    for i, (s, r, _, t) in enumerate(q[4:200]):
        np.testing.assert_array_equal(fi.col('objects')[b[i]:e[i]],
                                      np.unique(q[(q[:, 0] == s) & (q[:, 1] == r) & (q[:, 3] == t)][:, 2]))


# ---- the oracle -----------------------------------------------------------------------------------------------------------
def _filtered_rank(pred, label, known):
    """model.py:403-418 restated: torch.sigmoid, the known answers zeroed, the label's own score restored, then the tie rule
    #greater + (#equal - 1) / 2 + 1."""
    p = torch.sigmoid(torch.from_numpy(np.asarray(pred, dtype=np.float32)))
    ground = p[label].clone()
    p[torch.from_numpy(np.asarray(known, dtype=np.int64))] = 0
    p[label] = ground
    return float((p > ground).sum()) + (float((p == ground).sum()) - 1) / 2 + 1


def oracle_ranks():
    """From the unmodified reference's scores of the golden run (renet_eval_tiny.npz's sub_pred / ob_pred): the static
    filter restated (checked against the golden's filtered ranks) and the time-aware filter.  Returns (static, time-aware
    [n, 2] as [sub, ob] per test triple, keep: the triples other than the rolled-over one)."""
    ev, tiny = load_npz('renet_eval_tiny.npz'), load_npz('renet_tiny.npz')
    q = tiny['quads'].astype(np.int64)
    te = ev['te']
    static, timed = np.zeros((len(te), 2)), np.zeros((len(te), 2))
    for k, i in enumerate(te):
        s, r, o, t = q[i]
        for j, (pred, label, col_fix, col_out, fix) in enumerate(((ev['sub_pred'][k], s, 2, 0, o), (ev['ob_pred'][k], o, 0, 2, s))):
            same = (q[:, col_fix] == fix) & (q[:, 1] == r)
            static[k, j] = _filtered_rank(pred, label, q[same][:, col_out])
            timed[k, j] = _filtered_rank(pred, label, q[same & (q[:, 3] == t)][:, col_out])
    return static, timed, te != ev['rolled_at']


def test_oracle_restates_the_reference_filter():
    ev = load_npz('renet_eval_tiny.npz')
    static, timed, keep = oracle_ranks()
    assert keep.sum() == len(keep) - 1
    # the golden's filtered ranks of the rolled triple come from its re-bound scores, which the golden does not store
    np.testing.assert_array_equal(static[keep], ev['filt'][keep])
    assert (timed[keep] != static[keep]).any()                       # the time-aware filter changes some ranks here
    assert (timed[keep] >= static[keep]).all()                     # it removes a subset of the static filter's answers


# ---- the flow on a host model ---------------------------------------------------------------------------------------------
def _run(ctx, batched, te=None, raw=False, time_aware=True, seed=1234):
    m, quads, gm = ctx['model'], ctx['quads'], ctx['gm']
    S, ST, O, OT = ctx['hist']
    te = ctx['ev']['te'] if te is None else te
    m.latest_time = torch.tensor(int(quads[te[0], 3]))
    torch.manual_seed(seed)
    fn = m.evaluate_stream_batched if batched else m.evaluate_stream
    kw = {'time_aware': True} if time_aware else {}
    return fn(quads[te], ([S[i] for i in te], [ST[i] for i in te]), ([O[i] for i in te], [OT[i] for i in te]), gm,
              total_data=None if raw and not time_aware else quads, raw=raw, **kw)


def test_host_batched_time_aware_matches_oracle():
    ctx = _ctx()
    ev = ctx['ev']
    _, timed, keep = oracle_ranks()
    out = _run(ctx, True)
    pr = out['protocols']
    assert sorted(pr) == ['filtered', 'raw', 'time_filtered']
    k2 = np.repeat(keep, 2)
    np.testing.assert_array_equal(pr['time_filtered']['ranks'][k2], timed.reshape(-1)[k2])
    np.testing.assert_array_equal(pr['filtered']['ranks'], ev['filt'].reshape(-1))
    np.testing.assert_array_equal(pr['raw']['ranks'][k2], ev['raw'].reshape(-1)[k2])
    np.testing.assert_array_equal(out['ranks'], ev['filt'].reshape(-1))             # top level: raw=False selects filtered
    for name in pr:
        assert pr[name]['loss'] == out['loss']
        assert abs(pr[name]['mrr'] - np.mean(1.0 / pr[name]['ranks'])) < 1e-12
    assert rel_err(out['loss'], float(ev['loss'].sum())) < 1e-4
    assert pr['time_filtered']['mrr'] < pr['filtered']['mrr']


def test_evaluate_filter_time_matches_oracle():
    """The per-triple reference form: one predict per call, ranks against the same-timestamp answers."""
    ctx = _ctx()
    m, ev, quads, gm = ctx['model'], ctx['ev'], ctx['quads'], ctx['gm']
    S, ST, O, OT = ctx['hist']
    _, timed, keep = oracle_ranks()
    m.latest_time = torch.tensor(ctx['t_test'])
    torch.manual_seed(1234)
    calls = []
    orig = m.predict
    m.predict = lambda *a: calls.append(1) or orig(*a)
    with torch.no_grad():
        for k, i in enumerate(ev['te']):
            r, loss = m.evaluate_filter_time(torch.from_numpy(quads[i]), (S[i], ST[i]), (O[i], OT[i]), gm, quads)
            if keep[k]:
                np.testing.assert_array_equal(r, timed[k])
    assert len(calls) == len(ev['te'])


@pytest.mark.parametrize('rebinding', [True, False])
@pytest.mark.parametrize('raw', [True, False])
def test_host_batched_equals_per_triple_time_aware(rebinding, raw):
    """Three timestamps (two roll-overs): batched and per-triple give equal ranks under all three protocols and the same
    state, and their top-level keys equal the time_aware=False result."""
    a, b, c = _ctx(rebinding), _ctx(rebinding), _ctx(rebinding)
    quads, ev = a['quads'], a['ev']
    va_last = ev['va'][quads[ev['va'], 3] == quads[ev['va'], 3].max()]
    te = np.concatenate((va_last[:8], ev['te']))
    assert len(np.unique(quads[te, 3])) == 3
    ref = _run(a, False, te, raw)
    got = _run(b, True, te, raw)
    plain = _run(c, True, te, raw, time_aware=False)
    for name in ('raw', 'filtered', 'time_filtered'):
        np.testing.assert_array_equal(got['protocols'][name]['ranks'], ref['protocols'][name]['ranks'])
    assert rel_err(got['loss'], ref['loss']) < 1e-6
    _assert_same_state(_state(a), _state(b))
    _assert_same_state(_state(b), _state(c))
    assert 'protocols' not in plain
    for k in ('mrr', 'mr', 'hits@1', 'hits@3', 'hits@10', 'loss'):
        assert got[k] == plain[k], k
    np.testing.assert_array_equal(got['ranks'], plain['ranks'])
    np.testing.assert_array_equal(got['ranks'], got['protocols']['raw' if raw else 'filtered']['ranks'])


def test_time_aware_needs_quadruples():
    ctx = _ctx()
    quads = ctx['quads']
    for batched in (True, False):
        fn = ctx['model'].evaluate_stream_batched if batched else ctx['model'].evaluate_stream
        with pytest.raises(ValueError, match='quadruples'):
            fn(quads[:1], ([[]], [[]]), ([[]], [[]]), ctx['gm'], total_data=None, raw=True, time_aware=True)
        with pytest.raises(ValueError, match='time column'):
            fn(quads[:1], ([[]], [[]]), ([[]], [[]]), ctx['gm'], total_data=quads[:, :3], time_aware=True)


# ---- the kernel, without a GPU ----------------------------------------------------------------------------------------------
def test_rank_multi_epilogue_has_integer_atomics_only(sass):  # noqa: F811
    for name, body in _matching(sass, r'umma_gemm_packed_kernel<\(bool\)0, \(int\)7>').items():
        hits = [ln.strip() for ln in body.split('\n') if FLOAT_ATOMIC.search(ln)]
        assert not hits, '%s: %s' % (name, hits[:3])
        assert re.search(r'\b(RED|REDG|ATOM|ATOMG)\.E\.ADD', body), name


def test_decoder_rank_multi_rejects_bad_arguments():
    """Every case returns -1 with its message before anything is launched (the fake addresses are never dereferenced).  The
    library's last-error string is per thread: the calls run on a thread of their own and leave this one's empty."""
    from renet_b200 import _lib
    L = _lib.lib()
    f = _lib.ctypes.c_void_p(4096)
    cases = ((3, f, f, f, 8, 1 << 30, b'outside 0..2'),
             (-1, None, None, None, 8, 1 << 30, b'outside 0..2'),
             (1, None, f, f, 8, 1 << 30, b'needs excl_col'),
             (2, f, None, f, 8, 1 << 30, b'excl_begin and excl_end'),
             (1, f, f, None, 8, 1 << 30, b'excl_begin and excl_end'),
             (0, None, None, None, 6, 1 << 30, b'multiple of 4'),
             (2, f, f, f, 8, 16, b'workspace too small'))
    got = []

    def run():
        for n_lists, col, begin, end, K, ws, _ in cases:
            rc = L.renet_decoder_rank_multi(f, f, None, f, n_lists, col, begin, end, f, f, 4, 10, K, f, ws, None)
            got.append((rc, L.renet_last_error()))
    t = threading.Thread(target=run)
    t.start()
    t.join()
    assert len(got) == len(cases)
    for (rc, err), case in zip(got, cases):
        assert rc == -1 and case[-1] in err, (case, rc, err)
