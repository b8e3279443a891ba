"""-m gpu: batched test-time scoring -- the fused rank decoder (renet_decoder_rank) against fp64 PyTorch and against torch's own
counts on planted exact ties, grouped encoding against the per-query encode, pred_r_topk on isolation groups against the
per-entity graph copies it used before, and RENet.evaluate_stream_batched end to end against the goldens and side by side
with the per-triple evaluate_stream."""
import numpy as np
import pytest
import torch

from helpers import eval_setup, load_npz, rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


# ---- the kernel -------------------------------------------------------------------------------------------------------------
def _exclusions(rng, M, N, labels, kind='random'):
    lists = []
    for m in range(M):
        if kind == 'random':
            n = int(rng.choice([0, 1, 3, 20, 300]))
            c = np.unique(rng.randint(0, N, n))
            if m % 3 == 0:
                c = np.unique(np.concatenate((c, [labels[m]])))           # the label inside its own list
        lists.append(c)
    col = np.concatenate(lists).astype(np.int32) if lists else np.zeros(0, np.int32)
    end = np.cumsum([len(c) for c in lists])
    begin = end - np.asarray([len(c) for c in lists])
    return lists, tuple(torch.from_numpy(np.asarray(a, dtype=np.int32)).to(DEV) for a in (col, begin, end))


def _band(z64, labels, lists, eps):
    """Per row: raw and filtered (strictly greater, near) counts from fp64 logits.  A column is near when its logit lies
    within eps of the label's (raw) or when the fp32 sigmoid intervals of [z - eps, z + eps] touch (filtered)."""
    M = z64.shape[0]
    idx = torch.arange(M, device=z64.device)
    lab = torch.as_tensor(labels, device=z64.device)
    zl = z64[idx, lab].view(-1, 1)
    d = z64 - zl
    not_l = torch.ones_like(d, dtype=torch.bool)
    not_l[idx, lab] = False
    g_raw = (d > eps).sum(1)
    n_raw = ((d.abs() <= eps) & not_l).sum(1)
    lo, hi = torch.sigmoid((z64 - eps).float()), torch.sigmoid((z64 + eps).float())
    excl = torch.zeros_like(d, dtype=torch.bool)
    for m, c in enumerate(lists):
        if len(c):
            excl[m, torch.as_tensor(c, device=z64.device).long()] = True
    excl &= not_l
    lo = torch.where(excl, torch.zeros_like(lo), lo)
    hi = torch.where(excl, torch.zeros_like(hi), hi)
    llo, lhi = lo[idx, lab].view(-1, 1), hi[idx, lab].view(-1, 1)
    g_f = ((lo > lhi) & not_l).sum(1)
    n_f = (~(lo > lhi) & ~(hi < llo) & not_l).sum(1)
    return g_raw, n_raw, g_f, n_f


def _check_band(rank, g, n):
    rank, g, n = rank.cpu().double(), g.cpu().double(), n.cpu().double()
    exact = n == 0
    assert torch.equal(rank[exact], g[exact] + 1)
    assert bool(((rank >= g + 1) & (rank <= g + n + 1)).all())
    return int((~exact).sum())


@pytest.mark.parametrize('M,N,K', [(1, 23033, 600), (2920, 23033, 600), (1760, 7691, 600), (64, 457, 600), (129, 2000, 600)])
def test_decoder_rank_vs_fp64(M, N, K):
    from renet_b200.decoder import decoder_rank, decoder_rank_counts
    rng = np.random.RandomState(M + N)
    gen = torch.Generator().manual_seed(M * 7 + N)
    x = (torch.randn(M, K, generator=gen) * 0.3).to(DEV)
    w = (torch.randn(N, K, generator=gen) * 0.3 / K ** 0.5 * 4).to(DEV)
    b = (torch.randn(N, generator=gen) * 0.5).to(DEV)
    labels = rng.randint(0, N, M)
    fixed = [0, 199, 200, N - 1]
    labels[:min(M, 4)] = fixed[:min(M, 4)]
    lists, ex = _exclusions(rng, M, N, labels)
    lab = torch.from_numpy(labels).to(DEV)
    loss, raw, filt = decoder_rank(x, w, b, lab, ex)
    z64 = x.double() @ w.double().t() + b.double()
    ref_loss = torch.logsumexp(z64, 1) - z64[torch.arange(M, device=DEV), lab]
    assert rel_err(loss.cpu().numpy(), ref_loss.cpu().numpy()) < 1e-4
    eps = 1e-5                                   # the 3xTF32 logits' error here is of the order of 1e-6
    g_raw, n_raw, g_f, n_f = _band(z64, labels, lists, eps)
    in_band = _check_band(raw, g_raw, n_raw), _check_band(filt, g_f, n_f)
    print('M=%d N=%d: rows in the near-tie band raw %d, filtered %d of %d' % (M, N, in_band[0], in_band[1], M))
    l2, c2 = decoder_rank_counts(x, w, b, lab, ex)
    l3, c3 = decoder_rank_counts(x, w, b, lab, ex)
    assert torch.equal(l2, l3) and torch.equal(c2, c3) and torch.equal(l2, loss)
    assert bool((c2[:, 1] >= 1).all())                       # the label's own logit equals pass 1's bit for bit
    _, c_none = decoder_rank_counts(x, w, b, lab, None)
    assert torch.equal(c_none[:, :2], c2[:, :2]) and not c_none[:, 2:].any()


def test_decoder_rank_planted_exact_ties():
    """Small-integer X, W and b: the 3xTF32 logits are exact, so the counts must equal torch's on the same logits, with
    torch.sigmoid on the device: ties with the label, sigmoids saturated to 1.0, sigmoids of 0 tying with the excluded
    zeros, the label in its own list, lists across column tiles, a list of about half of N, and empty lists."""
    from renet_b200.decoder import decoder_rank_counts
    from renet_b200.inference import rank_counts_torch
    M, N, K = 10, 457, 8
    rng = np.random.RandomState(5)
    x = torch.from_numpy(rng.randint(-2, 3, (M, K)).astype(np.float32))
    w = torch.from_numpy(rng.randint(-2, 3, (N, K)).astype(np.float32))
    b = torch.from_numpy(rng.choice([-120.0, -100.0, 0.0, 1.0, 18.0, 20.0, 25.0], N).astype(np.float32))
    x, w, b = x.to(DEV), w.to(DEV), b.to(DEV)
    z = (x.double() @ w.double().t() + b.double()).float()
    p = torch.sigmoid(z)
    assert int((p == 1.0).sum()) > 50 and int((p == 0.0).sum()) > 50
    zero_col = int(torch.nonzero(p[6] == 0)[0])
    one_col = int(torch.nonzero(p[7] == 1)[0])
    labels = np.asarray([0, 199, 200, 456, 3, 17, zero_col, one_col, 399, 401])
    lists = [np.zeros(0, np.int64),                                            # empty
             np.asarray([5, 199, 300]),                                        # the label inside its list
             np.concatenate((np.arange(190, 215), np.arange(395, 410))),     # across the column tiles at 200 and 400
             np.arange(0, N, 2),                                               # about half of N
             np.flatnonzero(p[4].cpu().numpy() == 1.0)[:40],                 # saturated columns excluded
             np.zeros(0, np.int64),
             np.flatnonzero(p[6].cpu().numpy() > 0.5),                        # sigma(label) = 0: excluded zeros tie with it
             np.flatnonzero(p[7].cpu().numpy() < 1.0)[::3],
             np.arange(200, 457),
             np.asarray([401])]
    col = np.concatenate(lists).astype(np.int32)
    end = np.cumsum([len(c) for c in lists])
    ex = tuple(torch.from_numpy(np.asarray(a, dtype=np.int32)).to(DEV) for a in (col, end - [len(c) for c in lists], end))
    lab = torch.from_numpy(labels).to(DEV)
    _, got = decoder_rank_counts(x, w, b, lab, ex)
    ref = rank_counts_torch(z, lab, ex)
    assert torch.equal(got.long(), ref), (got, ref)
    assert int(ref[:, 1].max()) > 1 and int(ref[6, 3]) > len(lists[6]) and int(ref[7, 3]) > 1   # the ties are there
    _, none = decoder_rank_counts(x, w, b, lab, None)
    assert torch.equal(none[:, :2].long(), ref[:, :2]) and not none[:, 2:].any()


def test_decoder_rank_rejects_bad_arguments():
    from renet_b200 import _lib
    L = _lib.lib()
    fake = _lib.ctypes.c_void_p(4096)
    rc = L.renet_decoder_rank(fake, fake, None, fake, fake, None, None, fake, fake, 4, 10, 8, fake, 1 << 30, None)
    assert rc == -1 and b'excl_begin' in L.renet_last_error()
    rc = L.renet_decoder_rank(fake, fake, None, fake, None, None, None, fake, fake, 4, 10, 6, fake, 1 << 30, None)
    assert rc == -1 and b'multiple of 4' in L.renet_last_error()


# ---- grouped encoding and pred_r_topk ---------------------------------------------------------------------------------------
def test_grouped_encoding_equals_encode_one():
    from test_gpu_rollover_topk import NUM_R, _model, _stream
    quads = _stream()
    m, gm = _model(quads)
    with torch.no_grad():
        m._roll_over(torch.tensor(312), gm)                     # histories now end with the predicted graph of t = 288
    for subject in (True, False):
        hist = m.s_hist_test if subject else m.o_hist_test
        hist_t = m.s_hist_test_t if subject else m.o_hist_test_t
        with_pred = [e for e in range(len(hist)) if len(hist_t[e]) and hist_t[e][-1] == 288][:6]
        assert with_pred
        empty = [e for e in range(len(hist)) if len(hist[e]) == 0][:2]
        ents = np.asarray(with_pred + [0, 5, 5, 17, 123, 5] + empty)
        rels = np.asarray([(3 * i) % NUM_R for i in range(len(ents))])
        fives = np.flatnonzero(ents == 5)
        rels[fives[1]] = rels[fives[0]]                             # a repeated (entity, relation) query
        has = np.asarray([len(hist[e]) != 0 for e in ents])
        has[2] = False                                              # predict's own empty-history test
        with torch.no_grad():
            got = m._encode_queries(ents, rels, has, subject)
            for i, (e, r) in enumerate(zip(ents, rels)):
                if not has[i]:
                    assert not got[i].any()
                    continue
                ref = m._encode_one(int(e), int(r), hist[e], hist_t[e], subject)
                assert rel_err(got[i].cpu().numpy(), ref.cpu().numpy()) < 1e-4, (subject, e, r)


def test_pred_r_topk_bitwise_equals_per_entity_copies():
    """pred_r_topk on isolation groups against the construction it replaced, built here by hand: every entity gets its own
    copies of its history's graphs, under keys of its own."""
    from renet_b200.decoder import ORDER_INDEX, decoder_group_topk
    from renet_b200.hoststore import GraphStore, HistoryStore
    from test_gpu_rollover_topk import NUM_K, NUM_R, _model, _stream
    quads = _stream()
    m, gm = _model(quads)
    R, h = NUM_R, m.h_dim
    with torch.no_grad():
        m._roll_over(torch.tensor(312), gm)
    for subject in (True, False):
        hist = m.s_hist_test if subject else m.o_hist_test
        hist_t = m.s_hist_test_t if subject else m.o_hist_test_t
        with_pred = [e for e in range(m.in_dim) if len(hist_t[e]) and hist_t[e][-1] == 288][:4]
        others = [e for e in range(m.in_dim) if len(hist[e]) and e not in with_pred][:8]
        assert with_pred and len(others) >= 4
        ents = he = np.asarray(with_pred + others + [others[0]])         # an entity twice: two groups of its own
        wts = torch.rand(len(ents), generator=torch.Generator().manual_seed(3)) * 0.1 + 1e-3
        rel_embeds, reverse = m._direction(subject)
        span = max(len(hist_t[e]) for e in he)
        keys = [[j * span + i for i in range(len(hist_t[e]))] for j, e in enumerate(he)]
        graphs, glob = {}, {}
        for e, ks in zip(he, keys):
            for v, t in zip(ks, hist_t[e]):
                graphs[v], glob[v] = m.graph_dict[int(t)], m.global_emb[int(t)]
        gs = GraphStore(graphs)
        view = HistoryStore([hist[e] for e in he], keys, he, gs, dedupe=False).select(np.repeat(np.arange(len(he)), R))
        with torch.no_grad():
            sh, sq, hb = m.aggregator.encode(view, torch.from_numpy(np.repeat(he, R)).to(DEV),
                                             torch.arange(R, device=DEV).repeat(len(he)), m.ent_embeds, rel_embeds, gs, glob,
                                             reverse, m.encoder, m.encoder_r)
            idx = hb.sample_order(DEV)
            sh_v, sq_v = torch.empty_like(sh), torch.empty_like(sq)
            sh_v[idx], sq_v[idx] = sh, sq
            ent = m.ent_embeds[torch.from_numpy(he).to(DEV)]
            s_q = sq_v.view(len(he), R, h)[:, 0]
            p_r = torch.softmax(m.linear_r(torch.cat((ent, s_q), dim=1)), dim=1)
            row_w = (wts.to(DEV).view(-1, 1) * p_r).reshape(-1)
            x = torch.cat((ent.repeat_interleave(R, dim=0), sh_v, rel_embeds.repeat(len(he), 1)), dim=1)
            v_ref, i_ref = decoder_group_topk(x, m.linear.weight, m.linear.bias, row_w, R, NUM_K, ORDER_INDEX)
            v, i = m.pred_r_topk(ents, wts, NUM_K, subject=subject)
        assert torch.equal(i, i_ref) and torch.equal(v, v_ref), subject


# ---- end to end -------------------------------------------------------------------------------------------------------------
def _golden_batched_flow(raw):
    """evaluate_stream_batched on the kernels over the golden's test split, checked against the golden: ranks (filtered, or
    raw with ``raw``), loss, the roll-over's histories and predicted graph, and the global model's calls."""
    from renet_b200 import _lib
    ctx = eval_setup(DEV)
    m, ev, quads, gm = ctx['model'], ctx['ev'], ctx['quads'], ctx['gm']
    S, ST, O, OT = ctx['hist']
    te = ev['te']
    m.latest_time = torch.tensor(ctx['t_test'])
    torch.manual_seed(1234)
    n0 = _lib.launch_count()
    out = m.evaluate_stream_batched(quads[te], ([S[i] for i in te], [ST[i] for i in te]), ([O[i] for i in te], [OT[i] for i in te]),
                                    gm, total_data=None if raw else quads, raw=raw)
    assert _lib.launch_count() > n0
    if raw:
        # the golden's raw ranks come from a second call per triple that never rolls over (test_eval_batched_host.py): its
        # rolled-over triple is scored without the re-binding there, so that triple's two ranks are left out
        keep = np.repeat(te != ev['rolled_at'], 2)
        assert keep.sum() == len(keep) - 2
        np.testing.assert_array_equal(out['ranks'][keep], ev['raw'].reshape(-1)[keep])
    else:
        np.testing.assert_array_equal(out['ranks'], ev['filt'].reshape(-1))
    assert rel_err(out['loss'], float(ev['loss'].sum())) < 1e-4
    np.testing.assert_array_equal([len(x) for x in m.s_hist_test], ev['after_len_s'])
    np.testing.assert_array_equal([len(x) for x in m.o_hist_test], ev['after_len_o'])
    t_pred = ctx['t_test']
    rows = [np.concatenate([[e], r]) for e in range(len(m.s_hist_test))
            if len(m.s_hist_test_t[e]) and m.s_hist_test_t[e][-1] == t_pred
            for r in np.asarray(m.s_hist_test[e][-1]).reshape(-1, 2)]
    np.testing.assert_array_equal(np.unique(np.asarray(rows, dtype=np.int64).reshape(-1, 3), axis=0), ev['after_new_s_rows'])
    g = m.graph_dict[t_pred]
    np.testing.assert_array_equal(np.sort(g.ndata['id'].view(-1).numpy()), ev['pred_graph_nodes'])
    assert g.number_of_edges() == int(ev['pred_graph_num_edges'])
    np.testing.assert_array_equal(np.asarray(gm.calls, dtype=np.int64), ev['gm_calls'])


def test_batched_flow_on_the_kernels_matches_reference_golden():
    _golden_batched_flow(raw=False)


def test_batched_raw_flow_on_the_kernels_matches_reference_golden():
    """Raw batched evaluation: the rank pass with no exclusion list."""
    _golden_batched_flow(raw=True)


def test_batched_flow_with_the_global_model_matches_reference_golden():
    from oracle import restate
    from oracle.gen_golden import RENET_SHAPES, det_params
    from renet_b200 import synthetic
    from renet_b200.global_model import RENet_global
    from renet_b200.model import RENet
    from test_gpu_eval_global import _HostOutputs
    ev, tiny = load_npz('renet_eval_global.npz'), load_npz('renet_tiny.npz')
    quads = tiny['quads'].astype(np.int64)
    num_e, R, h, nb, seed, num_k = int(tiny['num_e']), int(tiny['R']), int(ev['h']), int(ev['nb']), int(ev['seed']), int(ev['num_k'])
    gshapes = {str(k): tuple(int(x) for x in v[:2] if x > 0) for k, v in zip(ev['gshape_keys'], ev['gshape_vals'])}
    gm = RENet_global(num_e, h, R, dropout=0, model=3, seq_len=10, num_k=num_k, maxpool=1)
    gm.load_state_dict(det_params(gshapes, seed + 1), strict=True)
    gm = gm.to(DEV).eval()
    m = RENet(num_e, h, R, dropout=0, model=0, seq_len=10, num_k=num_k, num_bases=nb)
    m.load_state_dict(det_params(RENET_SHAPES(num_e, h, R, nb), seed), strict=True)
    m = m.to(DEV).eval()
    gd = synthetic.build_graph_dict(quads, R)
    tr, va, te = ev['tr'], ev['va'], ev['te']
    with torch.no_grad():
        m.global_emb = gm.get_global_emb([int(t) for t in np.unique(quads[tr][:, 3])], gd)
    m.graph_dict = gd
    S, ST, O, OT = restate.build_history(quads, num_e)
    pick = lambda L, idx: [L[i] for i in idx]                                           # noqa: E731
    m.init_history(quads[tr], (pick(S, tr), pick(ST, tr)), (pick(O, tr), pick(OT, tr)),
                   quads[va], (pick(S, va), pick(ST, va)), (pick(O, va), pick(OT, va)),
                   quads[te], (pick(S, te), pick(ST, te)), (pick(O, te), pick(OT, te)))
    m.latest_time = torch.tensor(int(quads[te[0], 3]))
    torch.manual_seed(4321)
    out = m.evaluate_stream_batched(quads[te], (pick(S, te), pick(ST, te)), (pick(O, te), pick(OT, te)), _HostOutputs(gm),
                                    total_data=quads)
    assert len(out['ranks']) == len(ev['ranks'])
    assert abs(out['mrr'] - float(ev['mrr'])) < 5e-4, (out['mrr'], float(ev['mrr']))
    assert abs(out['mr'] - float(ev['mr'])) < 5e-2, (out['mr'], float(ev['mr']))
    for k, want in zip((1, 3, 10), ev['hits']):
        assert abs(out['hits@%d' % k] - float(want)) < 5e-4 + 1.0 / len(ev['ranks']), (k, out['hits@%d' % k], float(want))
    assert np.mean(out['ranks'] == ev['ranks']) > 0.98


def _icews18_stream():
    """An ICEWS18-shaped synthetic stream: training histories up to the last three timestamps, which are the test split (two
    roll-overs)."""
    from oracle.stub_global import StubGlobalModel
    from renet_b200 import synthetic
    from renet_b200.model import RENet
    tkg = synthetic.SyntheticTKG('icews18', seed=13, num_timestamps=10, h_dim=200)
    quads = tkg.quads
    times = np.unique(quads[:, 3])
    tr, te = np.flatnonzero(quads[:, 3] < times[-3]), np.flatnonzero(quads[:, 3] >= times[-3])
    S, ST, O, OT = synthetic.build_history(quads)
    models = []
    for _ in range(2):
        torch.manual_seed(0)
        m = RENet(tkg.num_e, 200, tkg.num_r, dropout=0, model=0, seq_len=10, num_k=200).to(DEV).eval()
        m.global_emb = dict(tkg.global_emb)
        m.graph_dict = dict(tkg.graph_dict)
        pick = lambda L, idx: [L[i] for i in idx]                                       # noqa: E731
        m.init_history(quads[tr], (pick(S, tr), pick(ST, tr)), (pick(O, tr), pick(OT, tr)), [], ([], []), ([], []),
                       quads[te], (pick(S, te), pick(ST, te)), (pick(O, te), pick(OT, te)))
        m.latest_time = torch.tensor(int(times[-3]))        # as test.py starts: the first test timestamp rolls nothing
        models.append((m, StubGlobalModel(tkg.num_e, 200, 29)))
    return quads, te, (S, ST, O, OT), models


def test_batched_flow_side_by_side_on_icews18_shape():
    from renet_b200.inference import FilterIndex
    quads, te, (S, ST, O, OT), ((m_ref, gm_ref), (m_new, gm_new)) = _icews18_stream()
    assert len(np.unique(quads[te, 3])) >= 3
    args = lambda: (quads[te], ([S[i] for i in te], [ST[i] for i in te]), ([O[i] for i in te], [OT[i] for i in te]))  # noqa: E731
    logits = []
    orig = m_ref.predict

    def keep(triplet, s_hist, o_hist, global_model):
        out = orig(triplet, s_hist, o_hist, global_model)
        logits.append((out[1].double(), out[2].double()))
        return out
    m_ref.predict = keep
    torch.manual_seed(77)
    ref = m_ref.evaluate_stream(*args(), gm_ref, total_data=quads)
    rng_ref = (torch.get_rng_state(), torch.cuda.get_rng_state())
    torch.manual_seed(77)
    got = m_new.evaluate_stream_batched(*args(), gm_new, total_data=quads)
    rng_new = (torch.get_rng_state(), torch.cuda.get_rng_state())
    assert torch.equal(rng_ref[0], rng_new[0]) and torch.equal(rng_ref[1], rng_new[1])
    assert gm_ref.calls == gm_new.calls
    assert int(m_ref.latest_time) == int(m_new.latest_time)
    for name in ('s_hist_test_t', 'o_hist_test_t', 's_his_cache_t', 'o_his_cache_t'):
        assert list(getattr(m_ref, name)) == list(getattr(m_new, name)), name
    for name in ('s_hist_test', 'o_hist_test', 's_his_cache', 'o_his_cache'):
        for a, b in zip(getattr(m_ref, name), getattr(m_new, name)):
            if isinstance(a, list):
                assert len(a) == len(b) and all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b)), name
            else:
                assert np.array_equal(np.asarray(a), np.asarray(b)), name
    assert sorted(m_ref.graph_dict) == sorted(m_new.graph_dict) and sorted(m_ref.global_emb) == sorted(m_new.global_emb)
    assert rel_err(got['loss'], ref['loss']) < 1e-4
    # ranks: equal outside the near-tie band of the per-triple path's own logits
    fi = FilterIndex(quads)
    n_band, ranks = 0, got['ranks'].reshape(-1, 2)
    for k, i in enumerate(te):
        s, r, o = (int(v) for v in quads[i, :3])
        sub, ob = logits[k]
        for j, (z, label, direction, fix) in enumerate(((sub, s, 'subjects', o), (ob, o, 'objects', s))):
            b, e = fi.ranges(direction, [fix], [r])
            lists = [fi.col(direction)[b[0]:e[0]]]
            z = z.view(1, -1)
            eps = 1e-5 * max(1.0, float(z.abs().max()))      # cuBLAS fp32 against 3xTF32 logits, and s_h to ~1e-6
            _, _, g_f, n_f = _band(z, [label], lists, eps)
            n_band += _check_band(torch.tensor([ranks[k, j]]), g_f, n_f)
    print('ICEWS18 shape: %d ranks, %d in the near-tie band' % (ranks.size, n_band))
