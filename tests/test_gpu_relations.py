"""-m gpu: the relation head's calls (evaluate_relations_observed, forecast_relations_observed, forecast_relations) on the
kernels.

* Against tests/golden/renet_relations_observed.npz (the reference's inp_r -> encoder_r -> linear_r per triple and direction
  over its own history, R = 6): raw, filtered and time-aware relation ranks exact, loss to 1e-4, top-k ids exact and values
  to 1e-4, with the known relations left out.
* On the ICEWS18-shaped split of test_gpu_eval_observed.py (R = 256, h = 200: two 200-column tiles of linear_r) against a
  per-query fp64 restatement (_encode_one's s_q, linear_r in fp64): ranks exact where no other relation lies within the
  measured tie band of the label's logit, top-k id sets exact outside the near-tie band, values to 1e-3 relative.  The rows
  are sampled so that labels and top-k answers fall in both column tiles, and every row carries a different entity or
  history, so a row or tile mix-up shows.
* forecast_relations on the tiny stream against a per-query restatement over the same roll-overs, and its end state
  against forecast's.
* process_group: over gloo (one GPU) and NCCL (world 2, skipped below two GPUs) every rank returns the one-process result
  bit for bit.
* The rank and top-k kernels ran: renet_decoder_rank_multi / renet_decoder_topk calls are counted, and ``linear_r.forward``
  raises (no logits are materialised with torch)."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from helpers import eval_setup, load_npz, rel_err
from test_eval_sharded_host import _free_port, _stream
from test_forecast_observed_host import check_against_scores
from test_gpu_eval_observed import _split
from test_relations_host import _allowed, _filtered_rank, _known_relations

from renet_b200.inference import OBSERVED_RANK_ROWS

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _no_torch_logits(monkeypatch, m, forbid=True):
    """Counts the decoder entry points' calls (rows per call) and, with ``forbid``, makes linear_r.forward raise."""
    from renet_b200 import decoder
    calls = {'rank': [], 'topk': []}

    def no_logits(*a, **kw):
        raise AssertionError('linear_r.forward called: logits materialised with torch')
    if forbid:
        monkeypatch.setattr(m.linear_r, 'forward', no_logits)
    rank, topk = decoder.decoder_rank_counts_multi, decoder.decoder_topk

    def counted_rank(x, w, *a, **kw):
        assert w is m.linear_r.weight
        calls['rank'].append(x.shape[0])
        return rank(x, w, *a, **kw)

    def counted_topk(x, w, *a, **kw):
        assert w is m.linear_r.weight
        calls['topk'].append(x.shape[0])
        return topk(x, w, *a, **kw)
    monkeypatch.setattr(decoder, 'decoder_rank_counts_multi', counted_rank)
    monkeypatch.setattr(decoder, 'decoder_topk', counted_topk)
    return calls


def _golden_split(ctx, rows):
    S, ST, O, OT = ctx['hist']
    return (ctx['quads'][rows], ([S[i] for i in rows], [ST[i] for i in rows]), ([O[i] for i in rows], [OT[i] for i in rows]))


def test_relation_kernels_match_reference_golden(monkeypatch):
    from renet_b200 import _lib, synthetic
    ctx = eval_setup(DEV)
    m, quads = ctx['model'], ctx['quads']
    gold = load_npz('renet_relations_observed.npz')
    rows, R = gold['rows'], m.num_rels
    gd, ge = synthetic.build_graph_dict(quads, ctx['dims'][1]), dict(m.global_emb)
    calls = _no_torch_logits(monkeypatch, m)
    n0 = _lib.launch_count()
    out = m.evaluate_relations_observed(*_golden_split(ctx, rows), gd, ge, total_data=quads, time_aware=True)
    assert _lib.launch_count() > n0
    assert calls['rank'] == [2 * len(rows)] and not calls['topk']
    for key, gk in (('raw', 'raw'), ('filtered', 'filt'), ('time_filtered', 'time_filt')):
        np.testing.assert_array_equal(out['protocols'][key]['ranks'], gold[gk].reshape(-1), err_msg=key)
    assert rel_err(out['loss'], float(gold['loss'].astype(np.float64).sum())) < 1e-4
    for subject, side in ((True, 's'), (False, 'o')):
        c = 0 if subject else 2
        q = np.stack((quads[rows, c], quads[rows, 3]), 1)
        hist = synthetic.observed_history(quads, q[:, 0], q[:, 1], subject)
        z = gold['z_' + side].astype(np.float64)
        for case, known in (('none', None), ('static', quads[:, :3]), ('time_aware', quads)):
            for k in (1, 3, R):
                calls['topk'].clear()
                vals, ids = m.forecast_relations_observed(q, hist, gd, ge, k=k, subject=subject, known=known,
                                                          time_aware=case == 'time_aware')
                assert calls['topk'] == [len(q)]
                assert vals.is_cuda and vals.dtype == torch.float32 and ids.dtype == torch.long
                assert check_against_scores(vals, ids, z, _allowed(quads, q, subject, case, R), k, 1e-5, 1e-4) == 0
                if case == 'none' and k == R:
                    np.testing.assert_array_equal(ids.cpu().numpy(), gold['topk_ids_' + side])
                    assert np.abs(vals.cpu().numpy() - gold['topk_vals_' + side]).max() <= 1e-4


def _restated_relation_logits(m, ents, hists, subjects, gd, ge):
    """z fp64 [n, R]: _encode_one's s_q over each row's own history (zero when empty), then linear_r in fp64."""
    W, b = m.linear_r.weight.double(), m.linear_r.bias.double()
    out = []
    with torch.no_grad():
        for e, (hl, ht), subject in zip(ents, hists, subjects):
            s_q = (torch.zeros(m.h_dim, device=DEV) if len(hl) == 0
                   else m._encode_one(int(e), 0, hl, ht, subject, gd, ge, relation=True))
            out.append((W @ torch.cat((m.ent_embeds[int(e)], s_q)).double() + b).cpu())
    return torch.stack(out).numpy()


def _rank_with_band(z, label, excluded):
    """The reference's rank (sigmoid with ``excluded`` zeroed, label kept; raw on the logits when excluded is None) and the
    number of admissible relations whose logit lies within 1e-6 max(1, |z|max) of the label's."""
    if excluded is None:
        rank = (z > z[label]).sum() + ((z == z[label]).sum() - 1.0) / 2 + 1
    else:
        rank = _filtered_rank(z, label, excluded)
    near = np.abs(z - z[label]) <= 1e-6 * max(1.0, float(np.abs(z).max()))
    near[label] = False
    if excluded is not None:
        near[excluded] = False
    return rank, int(near.sum())


def test_relations_observed_matches_per_triple_restatement_on_icews18_shape(monkeypatch):
    quads, te, args, m, _ = _split()
    q, sh, oh, gd, ge = args
    R = m.num_rels
    assert R > 200 and m.h_dim == 200                       # linear_r spans two 200-column tiles
    calls = _no_torch_logits(monkeypatch, m)
    out = m.evaluate_relations_observed(*args, total_data=quads, time_aware=True)
    assert sum(calls['rank']) == 2 * len(q) and max(calls['rank']) <= OBSERVED_RANK_ROWS
    rng = np.random.RandomState(6)
    hi = np.flatnonzero(q[:, 1] >= 200)                     # labels in the second column tile
    rows = np.unique(np.concatenate((rng.choice(len(q), 150, replace=False), rng.choice(hi, min(50, len(hi)), replace=False))))
    assert (q[rows, 1] >= 200).any() and (q[rows, 1] < 200).any()
    ents = np.concatenate((q[rows, 0], q[rows, 2]))
    hists = [(sh[0][i], sh[1][i]) for i in rows] + [(oh[0][i], oh[1][i]) for i in rows]
    subjects = [True] * len(rows) + [False] * len(rows)
    z = _restated_relation_logits(m, ents, hists, subjects, gd, ge)
    checked, skipped = 0, 0
    for key in ('raw', 'filtered', 'time_filtered'):
        got = out['protocols'][key]['ranks'].reshape(-1, 2)
        for j, i in enumerate(rows):
            for side, subject in ((0, True), (1, False)):
                zz = z[j + side * len(rows)]
                e, r, t = int(q[i, 0 if subject else 2]), int(q[i, 1]), int(q[i, 3])
                excluded = None if key == 'raw' else _known_relations(quads, e, subject, t if key == 'time_filtered' else None)
                rank, near = _rank_with_band(zz, r, excluded)
                if near:
                    skipped += 1
                    assert abs(got[i, side] - rank) <= near, (key, i, side)
                    continue
                assert got[i, side] == rank, (key, i, side, got[i, side], rank)
                checked += 1
    print('relation ranks vs restatement: %d checked exactly, %d within the tie band' % (checked, skipped))
    assert skipped <= checked // 20
    # the loss: the rows' cross-entropies in fp64 over every triple is too slow to restate; the sampled rows' sum is
    # checked through a split of just those rows
    sub = (q[rows], ([sh[0][i] for i in rows], [sh[1][i] for i in rows]), ([oh[0][i] for i in rows], [oh[1][i] for i in rows]),
           gd, ge)
    got_loss = m.evaluate_relations_observed(*sub, raw=True)['loss']
    zt = torch.from_numpy(z)
    lab = torch.from_numpy(np.concatenate((q[rows, 1], q[rows, 1])))
    ref_loss = float(torch.nn.functional.cross_entropy(zt, lab, reduction='sum'))
    assert rel_err(got_loss, ref_loss) < 1e-5


@pytest.mark.parametrize('subject', [True, False])
def test_forecast_relations_observed_matches_restatement_on_icews18_shape(subject, monkeypatch):
    quads, te, args, m, _ = _split()
    q, sh, oh, gd, ge = args
    hist = sh if subject else oh
    c = 0 if subject else 2
    queries = np.stack((q[:, c], q[:, 3]), 1)
    rows = np.sort(np.random.RandomState(8).choice(len(queries), 200, replace=False))
    z = _restated_relation_logits(m, queries[rows, 0], [(hist[0][i], hist[1][i]) for i in rows], [subject] * len(rows),
                                  gd, ge)
    eps = 1e-5 * max(1.0, float(np.abs(z).max()))
    calls = _no_torch_logits(monkeypatch, m)
    for case, known in (('none', None), ('static', quads[:, :3]), ('time_aware', quads)):
        k = 10
        vals, ids = m.forecast_relations_observed(queries, hist, gd, ge, k=k, subject=subject, known=known,
                                                  time_aware=case == 'time_aware')
        allowed = _allowed(quads, queries[rows], subject, case, m.num_rels)
        n_band = check_against_scores(vals[rows], ids[rows], z, allowed, k, eps, 1e-3, relative=True)
        print('forecast_relations_observed vs restatement (%s, %s): %d rows, %d in the near-tie band of %.2e; answers '
              'past column 200: %d' % ('subject' if subject else 'object', case, len(rows), n_band, eps,
                                       int((ids[rows] >= 200).sum())))
        assert n_band <= len(rows) // 10
    per = -(-len(queries) // OBSERVED_RANK_ROWS)
    assert len(calls['topk']) == 3 * per and sum(calls['topk']) == 3 * len(queries)
    assert (ids >= 200).any()                               # answers come from both column tiles


def _tiny_forecast_relations(ctx, subject, k, known, group=None):
    m, quads = ctx['model'], ctx['quads']
    te = _stream(ctx)
    q = np.stack((quads[te, 0 if subject else 2], quads[te, 3]), 1)
    m.latest_time = torch.tensor(int(q[0, 1]))
    torch.manual_seed(1234)
    return q, m.forecast_relations(q, ctx['gm'], k=k, subject=subject, known=known, process_group=group)


def _state_digest(ctx):
    m = ctx['model']
    st = [int(m.latest_time), list(ctx['gm'].calls), torch.get_rng_state(), sorted(int(t) for t in m.graph_dict)]
    for name in ('s_hist_test', 'o_hist_test', 's_hist_test_t', 'o_hist_test_t', 's_his_cache', 'o_his_cache'):
        st.append([[np.asarray(x).tolist() for x in h] if isinstance(h, list) else np.asarray(h).tolist()
                   for h in getattr(m, name)])
    return st


def _same_state(a, b):
    return all(torch.equal(x, y) if isinstance(x, torch.Tensor) else x == y for x, y in zip(a, b))


@pytest.mark.parametrize('subject', [True, False])
def test_forecast_relations_matches_restatement_and_leaves_forecasts_state(subject, monkeypatch):
    ctx, ref = eval_setup(DEV), eval_setup(DEV)
    m, quads, R = ctx['model'], ctx['quads'], ctx['model'].num_rels
    # the roll-over weighs its candidates with softmax(linear_r(...)) as pred_r_topk always has, so linear_r.forward stays
    calls = _no_torch_logits(monkeypatch, m, forbid=False)
    q, (vals, ids) = _tiny_forecast_relations(ctx, subject, 4, quads)
    assert len(calls['topk']) == len(np.unique(q[:, 1])) and sum(calls['topk']) == len(q)
    monkeypatch.undo()
    # the restatement: the same roll-overs (forecast over the same timestamps), then each query's s_q and linear_r in fp64
    mr = ref['model']
    te = _stream(ref)
    mr.latest_time = torch.tensor(int(q[0, 1]))
    torch.manual_seed(1234)
    z = []
    for t in np.unique(q[:, 1]):
        sel = np.flatnonzero(q[:, 1] == t)
        mr.forecast(np.stack((q[sel, 0], quads[te[sel], 1], q[sel, 1]), 1), ref['gm'], k=4, subject=subject, known=quads)
        hist, hist_t = (mr.s_hist_test, mr.s_hist_test_t) if subject else (mr.o_hist_test, mr.o_hist_test_t)
        for e in q[sel, 0]:
            e = int(e)
            z.append(_restated_relation_logits(mr, [e], [(hist[e], hist_t[e])], [subject], mr.graph_dict, mr.global_emb)[0])
    assert _same_state(_state_digest(ctx), _state_digest(ref))      # forecast_relations leaves forecast's state and RNG
    z = np.stack(z)
    assert check_against_scores(vals, ids, z, _allowed(quads, q, subject, 'static', R), 4, 1e-5, 1e-4) <= len(q) // 10


def _init(rank, world, port, backend):
    if backend == 'nccl':
        os.environ['CUDA_VISIBLE_DEVICES'] = str(rank)      # before CUDA starts in this process
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(0)
    if backend == 'nccl':
        dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', 0))
    else:
        dist.init_process_group('gloo', rank=rank, world_size=world)


def _sharded_worker(rank, world, port, backend, out):
    _init(rank, world, port, backend)
    try:
        res = {}
        for subject in (True, False):
            ctx = eval_setup('cuda:0')
            _, (v, i) = _tiny_forecast_relations(ctx, subject, 4, ctx['quads'], dist.group.WORLD)
            res[subject] = (v.cpu(), i.cpu(), _state_digest(ctx))
        out[rank] = res
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('backend', ['nccl', 'gloo'])
def test_sharded_forecast_relations_equals_single_process(backend):
    if backend == 'nccl' and torch.cuda.device_count() < 2:
        pytest.skip('NCCL sharding needs two GPUs')
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_sharded_worker, args=(2, _free_port(), backend, out), nprocs=2, join=True)
    res = dict(out)
    mgr.shutdown()
    for subject in (True, False):
        ctx = eval_setup(DEV)
        _, (v, i) = _tiny_forecast_relations(ctx, subject, 4, ctx['quads'])
        ref_state = _state_digest(ctx)
        for rank in range(2):
            gv, gi, state = res[rank][subject]
            assert torch.equal(gv, v.cpu()) and torch.equal(gi, i.cpu()), (backend, subject, rank)
            assert _same_state(state, ref_state), (backend, subject, rank)
