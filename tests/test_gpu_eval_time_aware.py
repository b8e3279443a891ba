"""-m gpu: the time-aware filter on the kernels -- renet_decoder_rank_multi (two exclusion lists in one counting pass) against
fp64 PyTorch, against torch's own counts on planted exact ties and against renet_decoder_rank; and
evaluate_stream_batched(time_aware=True) end to end against the oracle of test_eval_time_aware.py and side by side with the
per-triple evaluate_stream(time_aware=True)."""
import numpy as np
import pytest
import torch

from helpers import eval_setup, rel_err
from test_eval_time_aware import oracle_ranks
from test_gpu_eval_batched import _band, _check_band, _exclusions, _icews18_stream

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _multi_ranks(c, j):
    from renet_b200.decoder import ranks_from_counts
    return ranks_from_counts(c[:, 2 + 2 * j], c[:, 3 + 2 * j])


# ---- the kernel -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('M,N,K', [(1, 23033, 600), (2920, 23033, 600), (1760, 7691, 600), (64, 457, 600), (129, 2000, 600)])
def test_decoder_rank_multi_vs_fp64(M, N, K):
    from renet_b200.decoder import decoder_rank_counts, decoder_rank_counts_multi, ranks_from_counts
    rng = np.random.RandomState(M + N + 1)
    gen = torch.Generator().manual_seed(M * 5 + N)
    x = (torch.randn(M, K, generator=gen) * 0.3).to(DEV)
    w = (torch.randn(N, K, generator=gen) * 0.3 / K ** 0.5 * 4).to(DEV)
    b = (torch.randn(N, generator=gen) * 0.5).to(DEV)
    labels = rng.randint(0, N, M)
    labels[:min(M, 4)] = [0, 199, 200, N - 1][:min(M, 4)]
    lists_a, ex_a = _exclusions(rng, M, N, labels)                  # two independent lists per row, empty ones included
    lists_b, ex_b = _exclusions(rng, M, N, labels)
    lab = torch.from_numpy(labels).to(DEV)
    loss, c = decoder_rank_counts_multi(x, w, b, lab, [ex_a, ex_b])
    assert c.shape == (M, 6)
    z64 = x.double() @ w.double().t() + b.double()
    ref_loss = torch.logsumexp(z64, 1) - z64[torch.arange(M, device=DEV), lab]
    assert rel_err(loss.cpu().numpy(), ref_loss.cpu().numpy()) < 1e-4
    eps = 1e-5
    g_raw, n_raw, g_a, n_a = _band(z64, labels, lists_a, eps)
    _, _, g_b, n_b = _band(z64, labels, lists_b, eps)
    in_band = (_check_band(ranks_from_counts(c[:, 0], c[:, 1]), g_raw, n_raw), _check_band(_multi_ranks(c, 0), g_a, n_a),
               _check_band(_multi_ranks(c, 1), g_b, n_b))
    print('M=%d N=%d: rows in the near-tie band raw %d, list A %d, list B %d of %d' % (M, N, *in_band, M))
    # agreement with renet_decoder_rank, list by list, and reproducibility
    l1, c1 = decoder_rank_counts_multi(x, w, b, lab, [ex_a])
    l_ref, c_ref = decoder_rank_counts(x, w, b, lab, ex_a)
    assert torch.equal(l1, l_ref) and torch.equal(c1, c_ref)
    _, c_ref_b = decoder_rank_counts(x, w, b, lab, ex_b)
    assert torch.equal(c[:, :4], c1) and torch.equal(c[:, 4:], c_ref_b[:, 2:]) and torch.equal(loss, l1)
    l0, c0 = decoder_rank_counts_multi(x, w, b, lab, [])
    assert c0.shape == (M, 2) and torch.equal(c0, c1[:, :2]) and torch.equal(l0, l1)
    l2, c2 = decoder_rank_counts_multi(x, w, b, lab, [ex_a, ex_b])
    assert torch.equal(l2, loss) and torch.equal(c2, c)


def test_decoder_rank_multi_planted_exact_ties():
    """Small-integer operands: exact logits, so each list's pair equals torch's counts on that list -- ties with the label,
    saturated sigmoids, lists across the column tiles at 200 and 400, the label in its own list, empty lists."""
    from renet_b200.decoder import decoder_rank_counts_multi
    from renet_b200.inference import rank_counts_torch
    M, N, K = 10, 457, 8
    rng = np.random.RandomState(5)
    x = torch.from_numpy(rng.randint(-2, 3, (M, K)).astype(np.float32)).to(DEV)
    w = torch.from_numpy(rng.randint(-2, 3, (N, K)).astype(np.float32)).to(DEV)
    b = torch.from_numpy(rng.choice([-120.0, -100.0, 0.0, 1.0, 18.0, 20.0, 25.0], N).astype(np.float32)).to(DEV)
    z = (x.double() @ w.double().t() + b.double()).float()
    p = torch.sigmoid(z)
    assert int((p == 1.0).sum()) > 50 and int((p == 0.0).sum()) > 50
    labels = np.asarray([0, 199, 200, 456, 3, 17, int(torch.nonzero(p[6] == 0)[0]), int(torch.nonzero(p[7] == 1)[0]), 399, 401])
    pn = p.cpu().numpy()
    list_a = [np.zeros(0, np.int64), np.asarray([5, 199, 300]), np.concatenate((np.arange(190, 215), np.arange(395, 410))),
              np.arange(0, N, 2), np.flatnonzero(pn[4] == 1.0)[:40], np.zeros(0, np.int64), np.flatnonzero(pn[6] > 0.5),
              np.flatnonzero(pn[7] < 1.0)[::3], np.arange(200, 457), np.asarray([401])]
    list_b = [np.flatnonzero(pn[0] == 1.0), np.zeros(0, np.int64), np.arange(198, 203), np.arange(1, N, 2),
              np.zeros(0, np.int64), np.asarray([17, 18, 399, 400]), np.flatnonzero(pn[6] == 0.0)[:30],
              np.flatnonzero(pn[7] == 1.0), np.arange(0, 200), np.arange(390, 457)]

    def dev(lists):
        col = np.concatenate(lists).astype(np.int32)
        end = np.cumsum([len(c) for c in lists])
        return tuple(torch.from_numpy(np.asarray(a, dtype=np.int32)).to(DEV) for a in (col, end - [len(c) for c in lists], end))
    ex_a, ex_b = dev(list_a), dev(list_b)
    lab = torch.from_numpy(labels).to(DEV)
    _, got = decoder_rank_counts_multi(x, w, b, lab, [ex_a, ex_b])
    ref_a, ref_b = rank_counts_torch(z, lab, ex_a), rank_counts_torch(z, lab, ex_b)
    assert torch.equal(got[:, :4].long(), ref_a), (got, ref_a)
    assert torch.equal(got[:, 4:].long(), ref_b[:, 2:]), (got, ref_b)
    assert int(ref_a[:, 1].max()) > 1 and int(ref_a[6, 3]) > len(list_a[6]) and int(ref_a[7, 3]) > 1   # the ties are there
    assert int(ref_b[6, 3]) > 1 and int(ref_b[7, 3]) == 1         # list B of row 7 excludes every other saturated column


# ---- end to end -------------------------------------------------------------------------------------------------------------
def _golden_run(time_aware):
    ctx = eval_setup(DEV)
    m, ev, quads, gm = ctx['model'], ctx['ev'], ctx['quads'], ctx['gm']
    S, ST, O, OT = ctx['hist']
    te = ev['te']
    m.latest_time = torch.tensor(ctx['t_test'])
    torch.manual_seed(1234)
    kw = {'time_aware': True} if time_aware else {}
    out = m.evaluate_stream_batched(quads[te], ([S[i] for i in te], [ST[i] for i in te]), ([O[i] for i in te], [OT[i] for i in te]),
                                    gm, total_data=quads, **kw)
    state = {'rng': (torch.get_rng_state(), torch.cuda.get_rng_state()), 'gm_calls': list(gm.calls),
             'latest_time': int(m.latest_time)}
    for name in ('s_hist_test', 'o_hist_test', 's_hist_test_t', 'o_hist_test_t'):
        state[name] = [[np.asarray(x).tolist() for x in h] for h in getattr(m, name)]
    return out, state


def test_time_aware_flow_on_the_kernels_matches_oracle():
    from renet_b200 import _lib
    ev = eval_setup('cpu')['ev']
    _, timed, keep = oracle_ranks()
    n0 = _lib.launch_count()
    out, st = _golden_run(True)
    assert _lib.launch_count() > n0
    pr = out['protocols']
    k2 = np.repeat(keep, 2)
    np.testing.assert_array_equal(pr['time_filtered']['ranks'][k2], timed.reshape(-1)[k2])
    np.testing.assert_array_equal(pr['filtered']['ranks'], ev['filt'].reshape(-1))
    np.testing.assert_array_equal(pr['raw']['ranks'][k2], ev['raw'].reshape(-1)[k2])
    plain, st_plain = _golden_run(False)
    np.testing.assert_array_equal(out['ranks'], plain['ranks'])
    for k in ('mrr', 'mr', 'hits@1', 'hits@3', 'hits@10', 'loss'):
        assert out[k] == plain[k], k
    assert torch.equal(st['rng'][0], st_plain['rng'][0]) and torch.equal(st['rng'][1], st_plain['rng'][1])
    for k in st:
        if k != 'rng':
            assert st[k] == st_plain[k], k


def test_time_aware_side_by_side_on_icews18_shape():
    from renet_b200.inference import FilterIndex, TimeFilterIndex
    quads, te, (S, ST, O, OT), ((m_ref, gm_ref), (m_new, gm_new)) = _icews18_stream()
    args = lambda: (quads[te], ([S[i] for i in te], [ST[i] for i in te]), ([O[i] for i in te], [OT[i] for i in te]))  # noqa: E731
    logits = []
    orig = m_ref.predict

    def keep(triplet, s_hist, o_hist, global_model):
        out = orig(triplet, s_hist, o_hist, global_model)
        logits.append((out[1].double(), out[2].double()))
        return out
    m_ref.predict = keep
    torch.manual_seed(77)
    ref = m_ref.evaluate_stream(*args(), gm_ref, total_data=quads, time_aware=True)
    rng_ref = (torch.get_rng_state(), torch.cuda.get_rng_state())
    torch.manual_seed(77)
    got = m_new.evaluate_stream_batched(*args(), gm_new, total_data=quads, time_aware=True)
    rng_new = (torch.get_rng_state(), torch.cuda.get_rng_state())
    assert len(logits) == len(te)                                         # one predict per triple
    assert torch.equal(rng_ref[0], rng_new[0]) and torch.equal(rng_ref[1], rng_new[1])
    assert gm_ref.calls == gm_new.calls and int(m_ref.latest_time) == int(m_new.latest_time)
    for name in ('s_hist_test_t', 'o_hist_test_t', 's_his_cache_t', 'o_his_cache_t'):
        assert list(getattr(m_ref, name)) == list(getattr(m_new, name)), name
    for name in ('s_hist_test', 'o_hist_test', 's_his_cache', 'o_his_cache'):
        for a, b in zip(getattr(m_ref, name), getattr(m_new, name)):
            if isinstance(a, list):
                assert len(a) == len(b) and all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b)), name
            else:
                assert np.array_equal(np.asarray(a), np.asarray(b)), name
    assert rel_err(got['loss'], ref['loss']) < 1e-4
    for name in ('raw', 'filtered', 'time_filtered'):
        assert got['protocols'][name]['loss'] == got['loss']
    np.testing.assert_array_equal(got['ranks'], got['protocols']['filtered']['ranks'])
    # time-aware ranks: inside the near-tie band of the per-triple path's own logits, with the time-aware lists
    fi, tfi = FilterIndex(quads), TimeFilterIndex(quads)
    n_band, n_diff, ranks = 0, 0, got['protocols']['time_filtered']['ranks'].reshape(-1, 2)
    for k, i in enumerate(te):
        s, r, o, t = (int(v) for v in quads[i])
        sub, ob = logits[k]
        for j, (z, label, direction, fix) in enumerate(((sub, s, 'subjects', o), (ob, o, 'objects', s))):
            b, e = tfi.ranges(direction, [fix], [r], [t])
            lst = tfi.col(direction)[b[0]:e[0]]
            bs, es = fi.ranges(direction, [fix], [r])
            n_diff += not np.array_equal(lst, fi.col(direction)[bs[0]:es[0]])
            z = z.view(1, -1)
            eps = 1e-5 * max(1.0, float(z.abs().max()))
            _, _, g_f, n_f = _band(z, [label], [lst], eps)
            n_band += _check_band(torch.tensor([ranks[k, j]]), g_f, n_f)
    assert n_diff > 0
    print('ICEWS18 shape: %d time-aware ranks, %d in the near-tie band; %d rows with different static and time-aware lists'
          % (ranks.size, n_band, n_diff))
