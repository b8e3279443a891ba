"""-m gpu: RENet.forecast on the kernels, on the ICEWS18-shaped stream of test_gpu_eval_batched.py (trained-shape parameters,
three test timestamps, two roll-overs).

* It matches a per-query restatement (the same roll-overs, then _encode_one, ``linear``, softmax and the known answers
  taken out), with index sets exact outside the near-tie band of the restatement's own logits, in both directions, with
  the static and the time-aware filter.
* With no filter and k above the rank, each test triple's object sits at the place evaluate_stream_batched (raw,
  reference_rebinding=False) ranks it, on rows without ties; and the stream ends in the evaluation's state.
* Sharded over NCCL (two GPUs; skipped with fewer) and over gloo with both ranks on one GPU, every rank returns the
  single-process result bit for bit."""
import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_gpu_eval_batched import _icews18_stream
from test_gpu_eval_sharded import _digest, _free_port, _init

pytestmark = pytest.mark.gpu


def _queries(quads, te, subject):
    q = quads[te]
    return np.stack((q[:, 0] if subject else q[:, 2], q[:, 1], q[:, 3]), 1)


def _restated(m, gm, q, subject, known, time_aware, rows):
    """(z fp64 [len(rows), N], allowed bool [len(rows), N]) of the queries ``rows`` of q, rolling over as forecast does."""
    R = m.num_rels
    rel = m.rel_embeds[:R] if subject else m.rel_embeds[R:]
    hist, hist_t = (m.s_hist_test, m.s_hist_test_t) if subject else (m.o_hist_test, m.o_hist_test_t)
    fix, ans = (0, 2) if subject else (2, 0)
    m._trim_test_histories()
    zs, allowed = [], []
    with torch.no_grad():
        for j, (e, r, t) in enumerate(q):
            if int(m.latest_time) != int(t):
                m._roll_over(torch.tensor(int(t)), gm)
            if j not in rows:
                continue
            s_h = torch.zeros(m.h_dim, device='cuda') if len(hist[e]) == 0 else m._encode_one(int(e), int(r), hist[e], hist_t[e], subject)
            zs.append(m.linear(torch.cat((m.ent_embeds[int(e)], s_h, rel[int(r)]))).double().cpu())
            sel = (known[:, fix] == e) & (known[:, 1] == r)
            if time_aware:
                sel &= known[:, 3] == t
            a = np.ones(m.in_dim, bool)
            a[known[sel, ans]] = False
            allowed.append(a)
    return torch.stack(zs), np.stack(allowed)


@pytest.mark.parametrize('subject,time_aware', [(True, False), (False, True)])
def test_forecast_matches_per_query_restatement(subject, time_aware):
    quads, te, _, ((m_a, gm_a), (m_b, gm_b)) = _icews18_stream()
    q = _queries(quads, te, subject)
    k = 10
    torch.manual_seed(77)
    vals, ids = m_a.forecast(q, gm_a, k=k, subject=subject, known=quads, time_aware=time_aware)
    rows = set(np.random.RandomState(1).choice(len(q), min(600, len(q)), replace=False).tolist())
    torch.manual_seed(77)
    z, allowed = _restated(m_b, gm_b, q, subject, quads, time_aware, rows)
    assert _digest(m_a, gm_a.calls) == _digest(m_b, gm_b.calls)
    n_band = 0
    for j, row in enumerate(sorted(rows)):
        got = ids[row].cpu().numpy()
        assert (got >= 0).all() and allowed[j][got].all()
        zj = z[j]
        adm = np.flatnonzero(allowed[j])
        order = adm[np.argsort(-zj[adm].numpy(), kind='stable')]
        eps = 1e-5 * max(1.0, float(zj.abs().max()))             # cuBLAS fp32 against 3xTF32 logits, and s_h to ~1e-6
        if float(zj[order[k - 1]] - zj[order[k]]) <= eps:
            n_band += 1
            assert float(zj[got].min()) >= float(zj[order[k - 1]]) - eps
        else:
            assert set(got.tolist()) == set(order[:k].tolist()), row
        p = torch.softmax(zj, 0)[got]
        assert float(((vals[row].cpu().double() - p).abs() / p).max()) <= 1e-3, row
    assert n_band <= len(rows) // 20, n_band
    print('forecast vs restatement: %d rows, %d in the near-tie band' % (len(rows), n_band))


def test_label_sits_at_its_raw_rank_and_state_matches_evaluation():
    quads, te, (S, ST, O, OT), ((m_a, gm_a), (m_b, gm_b)) = _icews18_stream()
    for m in (m_a, m_b):
        m.reference_rebinding = False
    k = 2000
    torch.manual_seed(77)
    out = m_a.evaluate_stream_batched(quads[te], ([S[i] for i in te], [ST[i] for i in te]),
                                      ([O[i] for i in te], [OT[i] for i in te]), gm_a, raw=True)
    rng_a = (torch.get_rng_state(), torch.cuda.get_rng_state())
    torch.manual_seed(77)
    vals, ids = m_b.forecast(_queries(quads, te, True), gm_b, k=k)
    rng_b = (torch.get_rng_state(), torch.cuda.get_rng_state())
    assert torch.equal(rng_a[0], rng_b[0]) and torch.equal(rng_a[1], rng_b[1])
    assert _digest(m_a, gm_a.calls) == _digest(m_b, gm_b.calls)
    ob_rank = out['ranks'].reshape(-1, 2)[:, 1]
    ids, vals = ids.cpu().numpy(), vals.cpu().numpy()
    checked = 0
    for j, i in enumerate(te):
        # the evaluation scores a query with an empty caller history as empty: compare the rows both score alike
        if len(S[i]) == 0 or ob_rank[j] != int(ob_rank[j]) or ob_rank[j] > k:
            continue
        pos = int(ob_rank[j]) - 1
        v = vals[j]
        if (pos > 0 and v[pos - 1] == v[pos]) or (pos + 1 < k and v[pos + 1] == v[pos]):
            continue                                               # a tie in p: its order is by column
        assert ids[j, pos] == quads[i, 2], (j, pos)
        checked += 1
    assert checked >= 50, checked
    print('label positions checked: %d of %d triples' % (checked, len(te)))


# ---- sharded -------------------------------------------------------------------------------------------------------------
def _run(group=None):
    quads, te, _, ((m, gm), _) = _icews18_stream()
    torch.manual_seed(77)
    v, i = m.forecast(_queries(quads, te, False), gm, k=20, subject=False, known=quads, time_aware=True,
                      process_group=group)
    return dict(v=v.cpu(), i=i.cpu(), rng=(torch.get_rng_state(), torch.cuda.get_rng_state()), state=_digest(m, gm.calls))


def _worker(rank, world, port, backend, out):
    _init(rank, world, port, backend)
    try:
        out[rank] = _run(dist.group.WORLD)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('backend', ['nccl', 'gloo'])
def test_sharded_forecast_equals_single_process_bitwise(backend):
    if backend == 'nccl' and torch.cuda.device_count() < 2:
        pytest.skip('NCCL at world size 2 needs 2 GPUs')
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), backend, out), nprocs=2, join=True)
    res = dict(out)
    mgr.shutdown()
    ref = _run()
    for rank in range(2):
        got = res[rank]
        assert torch.equal(got['v'], ref['v']) and torch.equal(got['i'], ref['i']), rank
        assert torch.equal(got['rng'][0], ref['rng'][0]) and torch.equal(got['rng'][1], ref['rng'][1])
        assert got['state'] == ref['state']
