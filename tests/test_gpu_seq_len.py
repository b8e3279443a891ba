"""gpu: histories longer than 16 steps on the kernels.

  * the GRU C-ABI (renet_gru_fwd / _bwd, both dropout entries, the dense pair) at 17 to 80 steps, per row and per gradient
    row against fp64 autograd, with the recurrence that ran asserted from the launch count: the persistent kernel up to 64
    steps, the step loop above; and a workspace one float short of what max_len needs is refused before any launch;
  * the RE-Net training step (dropout off against fp64, dropout on bitwise reproducible) and the global model's
    pre-training step and embedding table at seq_len 20 and 32 at the ICEWS18 shape, per row against the fp64
    restatements; the global model and the test-time flow against the reference's
    seq_len = 20 golden;
  * evaluate_observed, forecast_observed and forecast_relations_observed on 32-step observed windows against a per-query
    fp64 restatement.
The bars are the encoder suite's (tests/encoder_contract_check.py): per row, |err|_inf <= tau (|ref row|_inf + 1e-2 |ref|_inf)
with tau = 1e-4 for states and 5e-4 for gradients."""
import numpy as np
import pytest
import torch

from encoder_contract_check import TAU_FWD, TAU_GRAD, row_ratio
from helpers import load_npz, rel_err
from oracle import restate

pytestmark = pytest.mark.gpu
dev = 'cuda:0'
F64 = torch.float64
PRELUDE = 15          # forward launches before the recurrence (tests/gru_contract_check.py), packed-weight cache off


def _ok(got, ref, tau, what):
    r = row_ratio(got.reshape(len(got), -1) if got.dim() > 1 else got.reshape(1, -1),
                  ref.reshape(len(ref), -1) if ref.dim() > 1 else ref.reshape(1, -1), tau)
    assert float(r.max()) <= 1.0, '%s: row %d is %.3g x the bar off' % (what, int(r.argmax()), float(r.max()))


# ---- the GRU C-ABI ----------------------------------------------------------------------------------------------------------
def _gru_case(L, mode, h=200, Q=300, T=37, short=False):
    from renet_b200 import _lib
    Lb, P = _lib.lib(), _lib.ptr
    torch.manual_seed(L)
    rng = np.random.RandomState(L)
    lens = np.sort(np.concatenate(([L] * 40, rng.randint(1, L + 1, Q - 40))))[::-1].astype(np.int64)
    S, max_len = int(lens.sum()), L
    bs = np.array([int((lens > t).sum()) for t in range(max_len)], dtype=np.int32)
    starts = np.concatenate(([0], np.cumsum(lens)[:-1])).astype(np.int32)
    dense, p_drop = mode == 'dense', (0.5 if mode == 'dropout' else 0.0)
    num_e, num_r, NH = 2000, 300, S // 2
    g = lambda *s, sc=1.0: torch.randn(*s, device=dev) * sc                                  # noqa: E731
    i32 = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.int32, device=dev)            # noqa: E731
    H2, ent, rel, glob = g(NH, h, sc=0.5), g(num_e, h, sc=0.3), g(num_r, h, sc=0.3), g(T, h, sc=0.1)
    readout = torch.randint(0, NH, (S,), device=dev, dtype=torch.int32)
    row_glob = torch.randint(0, T, (S,), device=dev, dtype=torch.int32)
    seq_s = torch.randint(0, num_e, (Q,), device=dev, dtype=torch.int32)
    seq_r = torch.randint(0, num_r, (Q,), device=dev, dtype=torch.int32)
    row_seq, seq_len, seq_start = i32(np.repeat(np.arange(Q), lens)), i32(lens), i32(starts)
    k4 = h if dense else 4 * h
    sc = 1.0 / h ** 0.5
    W = [g(3 * h, k4, sc=sc), g(3 * h, h, sc=sc), g(3 * h, sc=0.1), g(3 * h, sc=0.1),
         g(3 * h, 3 * h, sc=sc), g(3 * h, h, sc=sc), g(3 * h, sc=0.1), g(3 * h, sc=0.1)]
    X4d = g(S, k4, sc=0.5) if dense else None
    leaves = [t.double().requires_grad_(True) for t in [H2, ent, rel, glob] + W]
    H2r, entr, relr, globr, wi4, wh4, bi4, bh4, wi3, wh3, bi3, bh3 = leaves
    seed = 4242 + L
    if dense:
        X4r = X4d.double().requires_grad_(True)
        ref4, ref3 = restate.gru_final_hidden_batched(X4r, lens, wi4, wh4, bi4, bh4), None
    else:
        X4, X3, _, _ = restate.packed_inputs(H2r, readout.long(), lens, seq_s.long(), seq_r.long(), entr, relr,
                                             globr[row_glob.long()])
        if p_drop:
            m = torch.empty(S * 7 * h, device=dev)
            _lib.check(Lb.renet_dropout_mask(seed, 0, m.numel(), p_drop, P(m), _lib.stream()), 'renet_dropout_mask')
            X4, X3 = X4 * m[:S * 4 * h].view(S, 4 * h).double(), X3 * m[S * 4 * h:].view(S, 3 * h).double()
        ref4 = restate.gru_final_hidden_batched(X4, lens, wi4, wh4, bi4, bh4)
        ref3 = restate.gru_final_hidden_batched(X3, lens, wi3, wh3, bi3, bh3)
    dhn4, dhn3 = g(Q, h), (torch.zeros(Q, h, device=dev) if dense else g(Q, h))
    ((ref4 * dhn4.double()).sum() + (0 if dense else (ref3 * dhn3.double()).sum())).backward()

    hn4, hn3 = torch.full((Q, h), float('nan'), device=dev), torch.full((Q, h), float('nan'), device=dev)
    hbs = bs.ctypes.data_as(_lib.ctypes.c_void_p)
    wp = [P(t) for t in W]
    Tn = 1 if dense else T
    fbytes = int((Lb.renet_gru_workspace_bytes_len if mode == 'plain' else Lb.renet_gru_dropout_workspace_bytes_len)(
        S, Q, Tn, h, max_len))
    assert fbytes > int((Lb.renet_gru_workspace_bytes if mode == 'plain' else Lb.renet_gru_dropout_workspace_bytes)(S, Q, Tn, h))
    nbytes = fbytes - 4 if short else fbytes
    ws = torch.empty(fbytes // 4 + 32, device=dev)
    Lb.renet_set_weight_generation(-1)
    n0 = _lib.launch_count()
    st = _lib.stream()
    if dense:
        rc = Lb.renet_gru_dense_fwd(P(X4d), k4, None, 0, P(seq_len), P(seq_start), hbs, max_len, *wp[:4], None, None, None, None,
                                    P(hn4), P(hn3), S, Q, h, P(ws), nbytes, st)
    elif p_drop:
        rc = Lb.renet_gru_fwd_dropout(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel), P(row_seq), P(seq_s), P(seq_r),
                                      P(seq_len), P(seq_start), hbs, max_len, *wp, P(hn4), P(hn3), S, Q, T, h, p_drop, seed,
                                      P(ws), nbytes, st)
    else:
        rc = Lb.renet_gru_fwd(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel), P(seq_s), P(seq_r), P(seq_len),
                              P(seq_start), hbs, max_len, *wp, P(hn4), P(hn3), S, Q, T, h, P(ws), nbytes, st)
    launches = _lib.launch_count() - n0
    if short:
        torch.cuda.synchronize()
        assert rc == -1 and b'max_len' in Lb.renet_last_error(), (rc, Lb.renet_last_error())
        assert launches == 0 and torch.isnan(hn4).all(), 'a short workspace launched or wrote'
        return
    _lib.check(rc, 'gru forward')
    torch.cuda.synchronize()
    if mode == 'plain':
        if L <= 64:
            assert launches == PRELUDE + 1, '%d forward launches at %d steps, not the persistent recurrence' % (launches, L)
        else:
            assert launches >= PRELUDE + 2 * L - 1, '%d forward launches at %d steps, not the step loop' % (launches, L)
    _ok(hn4, ref4.detach(), TAU_FWD, 'hn4 at %d steps (%s)' % (L, mode))
    if not dense:
        _ok(hn3, ref3.detach(), TAU_FWD, 'hn3 at %d steps (%s)' % (L, mode))

    # backward: every output starts from a random base (accumulated) or NaN (written)
    ref_g = {'w_ih4': wi4.grad, 'w_hh4': wh4.grad, 'b_ih4': bi4.grad, 'b_hh4': bh4.grad}
    if not dense:
        ref_g.update({'d_ent': entr.grad, 'd_rel': relr.grad, 'd_glob': globr.grad, 'w_ih3': wi3.grad, 'w_hh3': wh3.grad,
                      'b_ih3': bi3.grad, 'b_hh3': bh3.grad})
    acc = {k: torch.randn_like(v.float()) for k, v in ref_g.items()}
    base = {k: v.clone() for k, v in acc.items()}
    wb = [P(t) for t in (W[0], W[1], W[4], W[5])]
    dw = [P(acc.get(k)) for k in ('w_ih4', 'w_hh4', 'b_ih4', 'b_hh4', 'w_ih3', 'w_hh3', 'b_ih3', 'b_hh3')]
    bfn = Lb.renet_gru_bwd_workspace_bytes_len if mode == 'plain' else Lb.renet_gru_bwd_dropout_workspace_bytes_len
    bbytes = int(bfn(S, Q, Tn, h, max_len))
    bws = torch.empty(bbytes // 4 + 32, device=dev)
    if dense:
        dX4 = torch.full((S, k4), float('nan'), device=dev)
        rc = Lb.renet_gru_dense_bwd(P(X4d), k4, None, 0, P(seq_len), P(seq_start), hbs, max_len, wb[0], wb[1], None, None,
                                    P(dhn4), P(dhn3), P(dX4), None, *dw[:4], None, None, None, None, S, Q, h, P(ws), P(bws),
                                    bbytes, st)
        written = {'dX4': (dX4, X4r.grad)}
    else:
        dH2 = torch.full((NH, h), float('nan'), device=dev)
        if p_drop:
            rc = Lb.renet_gru_bwd_dropout(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel), P(row_seq), P(seq_s),
                                          P(seq_r), P(seq_len), P(seq_start), hbs, max_len, *wb, P(dhn4), P(dhn3), P(dH2),
                                          P(acc['d_ent']), P(acc['d_rel']), P(acc['d_glob']), *dw, NH, S, Q, T, h, p_drop,
                                          seed, P(ws), P(bws), bbytes, st)
        else:
            rc = Lb.renet_gru_bwd(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel), P(seq_s), P(seq_r), P(seq_len),
                                  P(seq_start), hbs, max_len, *wb, P(dhn4), P(dhn3), P(dH2), P(acc['d_ent']),
                                  P(acc['d_rel']), P(acc['d_glob']), *dw, NH, S, Q, T, h, P(ws), P(bws), bbytes, st)
        written = {'dH2': (dH2, H2r.grad)}
    _lib.check(rc, 'gru backward')
    torch.cuda.synchronize()
    for k, (got, ref) in written.items():
        assert not torch.isnan(got).any(), k
        _ok(got, ref, TAU_GRAD, '%s at %d steps (%s)' % (k, L, mode))
    for k, ref in ref_g.items():
        _ok(acc[k].double() - base[k].double(), ref, TAU_GRAD, 'd%s at %d steps (%s)' % (k, L, mode))


@pytest.mark.parametrize('L', [17, 20, 32, 64, 80])
@pytest.mark.parametrize('mode', ['plain', 'dropout', 'dense'])
def test_gru_long_histories_against_fp64(L, mode):
    _gru_case(L, mode)


@pytest.mark.parametrize('mode', ['plain', 'dropout', 'dense'])
def test_gru_refuses_a_short_workspace(mode):
    _gru_case(20, mode, Q=64, short=True)


# ---- the training step ------------------------------------------------------------------------------------------------------
def _long_tkg(L, T=60):
    from renet_b200 import synthetic
    tkg = synthetic.SyntheticTKG('icews18', seed=7, num_timestamps=T)
    tkg.s_hist, tkg.s_hist_t, tkg.o_hist, tkg.o_hist_t = synthetic.build_history(tkg.quads, history_len=L)
    return tkg


@pytest.mark.parametrize('L', [20, 32])
def test_training_step_against_fp64(L):
    from renet_b200.model import RENet
    tkg = _long_tkg(L)
    q, sh, oh = tkg.batch(0, batch_size=256)
    assert max(len(x) for x in sh[0]) == L
    torch.manual_seed(0)
    m = RENet(tkg.num_e, 200, tkg.num_r, dropout=0, seq_len=L).to(dev).train()
    m.global_emb = tkg.global_emb
    batch = torch.from_numpy(q).long().to(dev)
    gd = restate.build_graph_dict(tkg.quads, tkg.num_r)
    glob = {t: v.double() for t, v in tkg.global_emb.items()}
    for subj, (H, HT) in ((True, sh), (False, oh)):
        m.zero_grad()
        loss = m(batch, sh, oh, tkg.graph_dict, subject=subj)
        loss.backward()
        P = {k: v.detach().cpu().double().requires_grad_(True) for k, v in m.state_dict().items()}
        ref = restate.renet_forward(P, q, H, HT, gd, glob, subj, tkg.num_r)
        assert len(ref['batch_sizes']) == L
        ref['loss'].backward()
        assert abs(loss.item() - ref['loss'].item()) <= 1e-5 * abs(ref['loss'].item())
        for k, p in m.named_parameters():
            if P[k].grad is not None:
                _ok(p.grad.cpu(), P[k].grad, TAU_GRAD, 'd%s at seq_len %d' % (k, L))


@pytest.mark.parametrize('L', [20, 32])
def test_training_step_with_dropout_is_reproducible(L):
    from renet_b200.model import RENet
    tkg = _long_tkg(L)
    q, sh, oh = tkg.batch(1, batch_size=512)
    batch = torch.from_numpy(q).long().to(dev)
    grads = []
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            torch.manual_seed(3)
            m = RENet(tkg.num_e, 200, tkg.num_r, dropout=0.5, seq_len=L).to(dev).train()
            m.global_emb = tkg.global_emb
            loss = m(batch, sh, oh, tkg.graph_dict, subject=True) + m(batch, sh, oh, tkg.graph_dict, subject=False)
            loss.backward()
            grads.append([loss.detach().clone()] + [p.grad.clone() for p in m.parameters() if p.grad is not None])
    finally:
        torch.use_deterministic_algorithms(prev)
    assert all(torch.isfinite(g).all() for g in grads[0])
    for a, b in zip(*grads):
        assert torch.equal(a, b)


# ---- the global model ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('L', [20, 32])
@pytest.mark.parametrize('pool', [1, 0])
def test_global_model_against_fp64(L, pool, monkeypatch):
    """The global model suite's restatement (tests/global_contract_check.py) at seq_len L: s_q rows, loss and every gradient
    row of both directions' pre-training step, the fp64 gradients routed through the kernel's layer-1 ReLU side and max-pool
    argmax as that suite routes them, and every row of the embedding table."""
    import global_contract_check as chk
    monkeypatch.setattr(chk, 'SEQ_LEN', L)
    s = chk.stream('icews18', L + 8, 11)
    sel = [L + 7, 0, 3, L + 2, L, 9]
    m = chk.make_model(s, pool, 0).train()
    t_list = np.asarray([s.times[i] for i in sel], dtype=np.int64)
    tp_s, tp_o = s.targets(sel)
    P = chk.params64(m)
    for rev in (False, True):
        tag = 'seq_len %d pool %d %s' % (L, pool, 'obj' if rev else 'subj')
        tp = tp_s if rev else tp_o
        st = chk.Step(s, t_list, rev)
        assert max(len(w) for w in st.wins) == L
        loss, sq, tgt, grads, rec = chk.run_step(m, s, t_list, tp_s, tp_o, rev)
        with torch.no_grad():
            ref_sq, ref_tgt, loss64 = st.forward(P, pool, tp)
        assert torch.equal(tgt, ref_tgt), tag
        chk.check_rows(tag, 's_q', sq[:st.Q], ref_sq)
        assert abs(float(loss) - float(loss64)) <= 1e-5 * abs(float(loss64)), (tag, float(loss), float(loss64))
        H2k, off, _ = rec['pool'][0]
        route = None
        if pool == 1:
            with torch.no_grad():
                _, H2r = chk.pooled64(P, s, st.uniq, rev, pool)
            route = chk.check_ties(tag, H2k.double(), H2r, off)
        _, _, lg = st.forward(P, pool, tp, times=st.uniq, route=route, mask1=rec['h1'][0] > 0)
        lin = 'linear_o' if rev else 'linear_s'
        keys = chk.GRAD_KEYS + [lin + '.weight', lin + '.bias']
        ref = dict(zip(keys, torch.autograd.grad(lg, [P[k] for k in keys], allow_unused=True)))
        chk.check_grads(tag, grads, {k: (g if g is not None else torch.zeros_like(P[k])) for k, g in ref.items()})
    m.eval()
    keys, queries = chk.table_queries(s, list(s.times))
    wins = [chk.window_of(s, q) for q in queries]
    assert max(len(w) for w in wins) == L
    with torch.no_grad():
        ref = chk.sq_of_windows(P, s, wins, False, pool)
        table = m.get_global_emb(list(s.times), s.gd)
    assert list(table) == keys
    chk.check_rows('seq_len %d pool %d table' % (L, pool), 'table', torch.cat([table[k].view(1, -1) for k in keys]), ref)


@pytest.mark.parametrize('pool', [1, 0])
def test_global_model_matches_reference_golden(pool):
    from oracle.gen_golden import det_params
    from renet_b200 import synthetic
    from renet_b200.global_model import RENet_global
    from test_seq_len_host import check_grad
    g = load_npz('renet_seq_len.npz')
    quads = g['quads'].astype(np.int64)
    num_e, R, seed = int(g['num_e']), int(g['R']), int(g['seed'])
    times = np.unique(quads[:, 3])
    gd = synthetic.build_graph_dict(quads, R)
    m = RENet_global(num_e, 200, R, seq_len=20, maxpool=pool)
    m.load_state_dict(det_params({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed + 5), strict=True)
    m = m.to(dev)
    sel = g['g_sel']
    for subj in (True, False):
        m.zero_grad()
        loss = m(torch.from_numpy(times[sel]), torch.from_numpy(g['true_prob_s'][sel]).to(dev),
                 torch.from_numpy(g['true_prob_o'][sel]).to(dev), gd, subject=subj)
        loss.backward()
        tag = 'pool%d/%s' % (pool, 'subj' if subj else 'obj')
        assert abs(loss.item() - float(g[tag + '/loss'])) < 1e-4 * abs(float(g[tag + '/loss']))
        for k, p in m.named_parameters():
            if p.grad is not None:
                assert check_grad(g, tag, k, p.grad.cpu().numpy()), (tag, k, 'not in the golden')
    if pool == 1:
        with torch.no_grad():
            ge = m.get_global_emb(times, gd)
        np.testing.assert_array_equal(list(ge), g['global_emb_keys'])
        assert rel_err(np.stack([v.view(-1).cpu().numpy() for v in ge.values()]), g['global_emb']) < 1e-4


# ---- evaluation -------------------------------------------------------------------------------------------------------------
def test_test_time_flow_matches_golden_and_batched_equals_stream():
    from test_eval_batched_host import _assert_same_state
    from test_seq_len_host import _eval_ctx, check_rolled_histories, run_test_split
    runs = []
    for batched in (False, True):
        m, g, quads, hist, gm = _eval_ctx()
        del m.aggregator.encode                                  # the kernels, not the oracle
        m.to(dev)
        out = run_test_split(m, g, quads, hist, gm, batched)
        np.testing.assert_array_equal(out['ranks'], g['filt'].reshape(-1))
        assert abs(out['loss'] - float(g['loss'].sum())) < 1e-4 * float(g['loss'].sum())
        check_rolled_histories(m, g)
        runs.append(_state_of(m, gm))
    _assert_same_state(*runs)


def _state_of(m, gm):
    st = {'latest_time': int(m.latest_time), 'gm_calls': list(gm.calls)}
    for name in ('s_hist_test', 'o_hist_test', 's_hist_test_t', 'o_hist_test_t', 's_his_cache', 'o_his_cache'):
        st[name] = [[np.asarray(x).tolist() for x in h] if isinstance(h, list) else np.asarray(h).tolist()
                    for h in getattr(m, name)]
    return st


def test_observed_calls_on_32_step_windows_against_fp64():
    from oracle.gen_golden import RENET_SHAPES, det_global_emb, det_params
    from renet_b200 import synthetic
    from renet_b200.inference import rank_with_ties
    from renet_b200.model import RENet
    L, h, nb, seed = 32, 8, 4, 9
    quads, num_e, R = synthetic.make_quads('tiny', seed=2, num_timestamps=L + 12)
    times = np.unique(quads[:, 3])
    gd, gd64 = synthetic.build_graph_dict(quads, R), restate.build_graph_dict(quads, R)
    glob = det_global_emb(times, h, seed + 1)
    params = det_params(RENET_SHAPES(num_e, h, R, nb), seed)
    m = RENet(num_e, h, R, seq_len=L, num_bases=nb)
    m.load_state_dict(params, strict=True)
    m = m.to(dev).eval()
    test = quads[quads[:, 3] >= times[-3]]
    sh = synthetic.observed_history(quads, test[:, 0], test[:, 3], True, history_len=L)
    oh = synthetic.observed_history(quads, test[:, 2], test[:, 3], False, history_len=L)
    assert max(len(x) for x in sh[0]) == L
    P = {k: v.double() for k, v in params.items()}
    glob64 = {t: v.double() for t, v in glob.items()}

    def states(ents, hist, subj):
        """fp64 s_h / s_q of each query alone (restate.renet_forward over a one-sample batch)."""
        s_h, s_q = torch.zeros(len(ents), h, dtype=F64), torch.zeros(len(ents), h, dtype=F64)
        for i, e in enumerate(ents):
            if len(hist[0][i]):
                tr = np.asarray([[e, test[i, 1], 0]] if subj else [[0, test[i, 1], e]])
                out = restate.renet_forward(P, tr, [hist[0][i]], [hist[1][i]], gd64, glob64, subj, R, nb)
                s_h[i], s_q[i] = out['s_h'][0], out['s_q'][0]
        return s_h, s_q

    sh_s, sq_s = states(test[:, 0], sh, True)
    sh_o, _ = states(test[:, 2], oh, False)
    ent = P['ent_embeds']
    z_o = torch.cat((ent[test[:, 0]], sh_s, P['rel_embeds'][:R][test[:, 1]]), 1) @ P['linear.weight'].t() + P['linear.bias']
    z_s = torch.cat((ent[test[:, 2]], sh_o, P['rel_embeds'][R:][test[:, 1]]), 1) @ P['linear.weight'].t() + P['linear.bias']
    with torch.no_grad():
        out = m.evaluate_observed(test, sh, oh, gd, glob, raw=True)
    ref = np.stack([[rank_with_ties(z_s[i], int(test[i, 0])), rank_with_ties(z_o[i], int(test[i, 2]))] for i in range(len(test))])
    np.testing.assert_array_equal(out['ranks'], ref.reshape(-1))
    ref_loss = float(torch.nn.functional.cross_entropy(z_o, torch.as_tensor(test[:, 2]), reduction='sum') +
                     torch.nn.functional.cross_entropy(z_s, torch.as_tensor(test[:, 0]), reduction='sum'))
    assert abs(out['loss'] - ref_loss) <= 1e-4 * abs(ref_loss)
    k = 5
    with torch.no_grad():
        vals, ids = m.forecast_observed(test[:, [0, 1, 3]], sh, gd, glob, k=k, subject=True)
        rvals, rids = m.forecast_relations_observed(test[:, [0, 3]], sh, gd, glob, k=k, subject=True)
    p = torch.softmax(z_o, 1)
    np.testing.assert_array_equal(ids.cpu().numpy(), torch.sort(p, dim=1, descending=True, stable=True).indices[:, :k].numpy())
    assert rel_err(vals.cpu().numpy(), torch.sort(p, dim=1, descending=True, stable=True).values[:, :k].numpy()) < 1e-4
    pr = torch.softmax(torch.cat((ent[test[:, 0]], sq_s), 1) @ P['linear_r.weight'].t() + P['linear_r.bias'], 1)
    np.testing.assert_array_equal(rids.cpu().numpy(), torch.sort(pr, dim=1, descending=True, stable=True).indices[:, :k].numpy())
    assert rel_err(rvals.cpu().numpy(), torch.sort(pr, dim=1, descending=True, stable=True).values[:, :k].numpy()) < 1e-4
