"""not gpu: host logic of RENet.evaluate_stream_batched (renet_b200/inference.py) against the reference's golden run and the
per-triple path, with the CPU oracle standing in for the CUDA encode as in test_inference_host.py; and the filter index
against evaluate_filter's masks."""
import numpy as np
import pytest
import torch

from helpers import eval_setup, rel_err
from test_inference_host import _oracle_encode


def _ctx(rebinding=True):
    ctx = eval_setup('cpu')
    ctx['model'].aggregator.encode = _oracle_encode(ctx)
    ctx['model'].reference_rebinding = rebinding
    return ctx


def _run(ctx, batched, te=None, raw=False, seed=1234):
    m, quads, gm = ctx['model'], ctx['quads'], ctx['gm']
    S, ST, O, OT = ctx['hist']
    te = ctx['ev']['te'] if te is None else te
    m.latest_time = torch.tensor(int(quads[te[0], 3]))
    torch.manual_seed(seed)
    fn = m.evaluate_stream_batched if batched else m.evaluate_stream
    return fn(quads[te], ([S[i] for i in te], [ST[i] for i in te]), ([O[i] for i in te], [OT[i] for i in te]), gm,
              total_data=None if raw else quads, raw=raw)


def _state(ctx):
    m = ctx['model']
    st = {'latest_time': int(m.latest_time), 'gm_calls': list(ctx['gm'].calls), 'rng': torch.get_rng_state(),
          'graph_keys': sorted(int(k) for k in m.graph_dict.keys()), 'glob_keys': sorted(int(k) for k in m.global_emb.keys())}
    for name in ('s_hist_test', 'o_hist_test', 'o_hist_test_t', 's_hist_test_t', 's_his_cache', 'o_his_cache'):
        st[name] = [[np.asarray(x).tolist() for x in h] if isinstance(h, list) else np.asarray(h).tolist()
                    for h in getattr(m, name)]
    st['s_his_cache_t'] = list(m.s_his_cache_t)
    g = m.graph_dict[int(m.latest_time)]
    st['graph'] = (np.sort(g.ndata['id'].view(-1).numpy()).tolist(), int(g.number_of_edges()))
    return st


def _assert_same_state(a, b):
    for k in a:
        if k == 'rng':
            assert torch.equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k


def test_batched_flow_matches_reference_golden():
    ctx = _ctx()
    ev, m = ctx['ev'], ctx['model']
    for k in ('hist_len_s', 'hist_len_o'):
        got = np.array([len(x) for x in (m.s_hist_test if k.endswith('s') else m.o_hist_test)])
        np.testing.assert_array_equal(got, ev[k])
    out = _run(ctx, True)
    np.testing.assert_array_equal(out['ranks'], ev['filt'].reshape(-1))                 # filtered ranks: exact
    assert rel_err(out['loss'], float(ev['loss'].sum())) < 1e-4
    t_test = int(ctx['quads'][ev['rolled_at'], 3])
    assert int(m.latest_time) == t_test
    np.testing.assert_array_equal([len(x) for x in m.s_hist_test], ev['after_len_s'])
    np.testing.assert_array_equal([len(x) for x in m.o_hist_test], ev['after_len_o'])
    t_pred = ctx['t_test']                                    # the roll-over predicts the graph of the previous timestamp
    rows = [np.concatenate([[e], r]) for e in range(len(m.s_hist_test))
            if len(m.s_hist_test_t[e]) and m.s_hist_test_t[e][-1] == t_pred
            for r in np.asarray(m.s_hist_test[e][-1]).reshape(-1, 2)]
    np.testing.assert_array_equal(np.unique(np.asarray(rows, dtype=np.int64).reshape(-1, 3), axis=0), ev['after_new_s_rows'])
    g = m.graph_dict[t_pred]
    np.testing.assert_array_equal(np.sort(g.ndata['id'].view(-1).numpy()), ev['pred_graph_nodes'])
    assert g.number_of_edges() == int(ev['pred_graph_num_edges'])
    np.testing.assert_array_equal(np.asarray(ctx['gm'].calls, dtype=np.int64), ev['gm_calls'])


def test_batched_raw_ranks_match_reference_golden():
    ctx = _ctx()
    ev = ctx['ev']
    out = _run(ctx, True, raw=True)
    # the golden's raw ranks come from a second call per triple (after the filtered one), which never rolls over: its
    # rolled-over triple is scored without the re-binding there, so that triple's two ranks are left out
    keep = np.repeat(ev['te'] != ev['rolled_at'], 2)
    assert keep.sum() == len(keep) - 2
    np.testing.assert_array_equal(out['ranks'][keep], ev['raw'].reshape(-1)[keep])


@pytest.mark.parametrize('rebinding', [True, False])
@pytest.mark.parametrize('raw', [True, False])
def test_batched_equals_per_triple_path(rebinding, raw):
    """Same ranks, loss and state as evaluate_stream, with and without the reference's re-binding, over a stream of three
    timestamps (two roll-overs)."""
    a, b = _ctx(rebinding), _ctx(rebinding)
    quads, ev = a['quads'], a['ev']
    va_last = ev['va'][quads[ev['va'], 3] == quads[ev['va'], 3].max()]
    te = np.concatenate((va_last[:8], ev['te']))               # the last validation timestamp, then the test split
    assert len(np.unique(quads[te, 3])) == 3
    ref = _run(a, False, te, raw)
    got = _run(b, True, te, raw)
    np.testing.assert_array_equal(got['ranks'], ref['ranks'])
    assert rel_err(got['loss'], ref['loss']) < 1e-6
    for k in ('mrr', 'mr', 'hits@1', 'hits@3', 'hits@10'):
        assert got[k] == ref[k], k
    _assert_same_state(_state(a), _state(b))


def test_filter_index_matches_evaluate_filter_masks():
    from renet_b200.inference import FilterIndex
    rng = np.random.RandomState(3)
    trip = np.stack((rng.randint(0, 30, 800), rng.randint(0, 6, 800), rng.randint(0, 30, 800)), 1)
    trip = np.concatenate((trip, trip[:100]))                                  # duplicates
    fi = FilterIndex(trip)
    allt = torch.from_numpy(trip)
    q = np.stack((rng.randint(0, 32, 300), rng.randint(0, 6, 300), rng.randint(0, 32, 300)), 1)
    for direction, col_fix, col_out, fix_col in (('objects', 0, 2, 0), ('subjects', 2, 0, 2)):
        b, e = fi.ranges(direction, q[:, fix_col], q[:, 1])
        col = fi.col(direction)
        assert col.dtype == np.int32
        for i, (s, r, o) in enumerate(q):
            fix = (s, r, o)[fix_col]
            known = allt[(allt[:, col_fix] == fix) & (allt[:, 1] == r)][:, col_out]
            np.testing.assert_array_equal(col[b[i]:e[i]], np.unique(known.numpy()))
