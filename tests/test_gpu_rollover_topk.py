"""-m gpu: the test-time roll-over's batched candidate scoring.

renet_decoder_group_topk (decoder.decoder_group_topk) against an fp64 PyTorch restatement of
    p[m, n] = w_m * softmax(x @ W^T + b)[m, n],   per group of R rows: the k largest p and their flat indices r * N + n,
with planted ties, the two output orders compared with torch.topk(sorted=False) itself, bitwise repeatability and the
capacity retry; then RENet.pred_r_topk and the roll-over against the per-entity pred_r_rank2 loop they replace
(reference model.py:222-279)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _fixture(G, R, N, K, seed, zscale=3.0):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(G * R, K, generator=gen)
    w = torch.randn(N, K, generator=gen) * (zscale / K ** 0.5)
    b = torch.randn(N, generator=gen) * 0.5
    rw = torch.rand(G * R, generator=gen) * 0.9 + 0.1
    return x, w, b, rw


def _reference(x, w, b, rw, R):
    """fp64 joint probabilities, one row of R * N per group."""
    z = x.double() @ w.double().t() + b.double()
    p = rw.double()[:, None] * torch.softmax(z, dim=1)
    return p.view(-1, R * w.shape[0])


def _torch_order(R, N):
    """The layout torch.topk(sorted=False) gives on CUDA, at every size used here (R * N from 40 to 5.9 M)."""
    from renet_b200.decoder import ORDER_INDEX
    return ORDER_INDEX


def _check_layout(values, indices, order):
    """A group's k entries are laid out as the order says (ties at the k-th value already went to the lower index)."""
    from renet_b200.decoder import ORDER_VALUE
    for v, i in zip(values.cpu(), indices.cpu()):
        if order == ORDER_VALUE:
            key = sorted(range(len(v)), key=lambda j: (-float(v[j]), int(i[j])))
        else:
            kth = float(v.min())
            key = sorted(range(len(v)), key=lambda j: (float(v[j]) == kth, int(i[j])))
        assert key == list(range(len(v)))


def _check_as_torch_topk(values, indices, R, N):
    """torch.topk(sorted=False) on a CUDA tensor of R * N values holding exactly these winners returns them in this order."""
    for v, i in zip(values, indices):
        q = torch.zeros(R * N, device=DEV)
        q[i] = v
        tv, ti = torch.topk(q, v.numel(), sorted=False)
        assert torch.equal(ti, i) and torch.equal(tv, v)


SHAPES = [(3, 1, 1000, 64, 10),            # R = 1
          (4, 8, 1001, 200, 50),           # N not a multiple of the 200-column tile
          (3, 2, 150, 24, 20),             # R * n_part = 4 < k: the threshold is 0, every entry is a candidate
          (2, 256, 23033, 600, 1),         # ICEWS18: R = 256 relations, |E| = 23 033, K = 3h
          (2, 256, 23033, 600, 10),
          (2, 256, 23033, 600, 1000)]


@pytest.mark.parametrize('G,R,N,K,k', SHAPES)
def test_group_topk_vs_fp64(G, R, N, K, k):
    from renet_b200.decoder import decoder_group_topk
    x, w, b, rw = _fixture(G, R, N, K, seed=G * 7 + R + N + K)
    ref = _reference(x.to(DEV), w.to(DEV), b.to(DEV), rw.to(DEV), R)
    rv, ri = torch.sort(ref, dim=1, descending=True, stable=True)
    # the index sets are well defined: the k-th and (k+1)-th fp64 values differ by more than 1e-5 relative
    if k < R * N:
        assert bool(((rv[:, k - 1] - rv[:, k]) > 1e-5 * rv[:, k - 1]).all()), 'fixture has a near tie at the k-th value'
    order = _torch_order(R, N)
    xs, ws, bs, rws = (t.to(DEV) for t in (x, w, b, rw))
    runs = [decoder_group_topk(xs, ws, bs, rws, R, k, order) for _ in range(2)]
    vals, idx = runs[0]
    assert vals.shape == (G, k) and idx.shape == (G, k) and idx.dtype == torch.int64
    for g in range(G):
        assert set(idx[g].tolist()) == set(ri[g, :k].tolist())
    got = ref.gather(1, idx)
    # the 3xTF32 logits: 4.4e-5 relative at most here, where the logits reach |z| = 17 (H100)
    assert float(((vals.double() - got).abs() / got).max()) <= 1e-4
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])       # bitwise repeatable
    _check_layout(vals, idx, order)
    _check_as_torch_topk(vals, idx, R, N)
    from renet_b200.decoder import ORDER_VALUE          # the same winners by value, ties by index
    v2, i2 = decoder_group_topk(xs, ws, bs, rws, R, k, ORDER_VALUE)
    assert all(set(a.tolist()) == set(c.tolist()) for a, c in zip(i2, idx))
    _check_layout(v2, i2, ORDER_VALUE)


@pytest.mark.parametrize('G,R,N,K,k', [SHAPES[1], SHAPES[5]])
def test_group_topk_capacity_retry(G, R, N, K, k):
    """A candidate buffer too small for a group is reported, never truncated; the wrapper repeats the call with the size
    reported and returns what a large enough buffer gives."""
    from renet_b200 import _lib
    from renet_b200.decoder import decoder_group_topk
    x, w, b, rw = (t.to(DEV) for t in _fixture(G, R, N, K, seed=5))
    order = _torch_order(R, N)
    L, P = _lib.lib(), _lib.ptr
    vals = torch.empty(G, k, device=DEV)
    idx = torch.empty(G, k, dtype=torch.int32, device=DEV)
    needed = torch.zeros(1, dtype=torch.int32, device=DEV)
    nbytes = int(L.renet_decoder_group_topk_workspace_bytes(G, R, N, K, k))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    _lib.check(L.renet_decoder_group_topk(P(x), P(w), P(b), P(rw), G, R, N, K, k, order, k, P(vals), P(idx), P(needed), P(ws),
                                          nbytes, _lib.stream()), 'renet_decoder_group_topk')
    assert int(needed.item()) > k
    small = decoder_group_topk(x, w, b, rw, R, k, order, capacity=k)
    full = decoder_group_topk(x, w, b, rw, R, k, order, capacity=R * N)
    assert torch.equal(small[0], full[0]) and torch.equal(small[1], full[1])


@pytest.mark.parametrize('R,N,k', [(4, 500, 2), (4, 500, 3), (64, 2000, 5)])
def test_group_topk_planted_ties(R, N, k):
    """Duplicated rows of W give bitwise equal logits: the winners at the k-th value are the lowest flat indices."""
    from renet_b200.decoder import decoder_group_topk
    G, K = 1, 40
    x, w, b, rw = _fixture(G, R, N, K, seed=11)
    rw[:] = 0.01
    rw[0] = 1.0                                          # row 0 dominates the group
    z0 = x[0].double() @ w.double().t() + b.double()
    top = int(torch.argmax(z0))
    twins = sorted({3, N // 2, N - 1} - {top})
    for c in twins:                                      # columns with row 0's top logit: ties at the top of the group
        w[c], b[c] = w[top], b[top]
    cols = sorted([top] + twins)
    order = _torch_order(R, N)
    vals, idx = decoder_group_topk(*(t.to(DEV) for t in (x, w, b, rw)), R, k, order)
    n_tied = min(k, len(cols))
    assert idx[0, :n_tied].tolist() == cols[:n_tied]     # the lowest indices of the tied entries, in index order
    assert bool((vals[0, :n_tied] == vals[0, 0]).all())
    _check_layout(vals, idx, order)
    _check_as_torch_topk(vals, idx, R, N)


def test_group_topk_rejects_bad_arguments():
    from renet_b200 import _lib
    from renet_b200.decoder import decoder_group_topk
    x, w, b, rw = (t.to(DEV) for t in _fixture(2, 4, 30, 8, seed=1))
    with pytest.raises(RuntimeError, match='outside'):
        decoder_group_topk(x, w, b, rw, 4, 4 * 30 + 1)             # k > R * N (torch.topk raises too)
    x6 = torch.randn(8, 6, device=DEV)
    with pytest.raises(RuntimeError, match='multiple of 4'):
        decoder_group_topk(x6, torch.randn(30, 6, device=DEV), b, rw, 4, 3)
    assert _lib.lib().renet_last_error()


# ---- RENet.pred_r_topk and the roll-over against the per-entity loop -------------------------------------------------------
NUM_E, NUM_R, H, NB, NUM_K = 300, 32, 16, 4, 50


def _stream():
    """A seeded stream of 15 timestamps over 32 relations and entities 0-249 with power-law popularity; entities 250-299
    never occur, so their histories stay empty."""
    rng = np.random.RandomState(3)
    n_seen = 250
    p_e = 1.0 / (np.arange(1, n_seen + 1) + 4.0) ** 1.3
    p_e /= p_e.sum()
    perm = rng.permutation(n_seen)
    out = []
    for ti in range(15):
        n = 160
        s = perm[rng.choice(n_seen, n, p=p_e)]
        o = perm[rng.choice(n_seen, n, p=p_e)]
        o[s == o] = (o[s == o] + 1) % n_seen
        r = rng.randint(0, NUM_R, n)
        out.append(np.stack((s, r, o, np.full(n, ti * 24)), axis=1))
    return np.concatenate(out).astype(np.int64)


def _model(quads):
    from oracle.stub_global import StubGlobalModel
    from renet_b200 import synthetic
    from renet_b200.model import RENet
    torch.manual_seed(0)
    m = RENet(NUM_E, H, NUM_R, dropout=0, model=0, seq_len=10, num_k=NUM_K, num_bases=NB)
    gen = torch.Generator().manual_seed(1)
    with torch.no_grad():                                # spread the scores: well separated top-k lists
        for p in m.parameters():
            p.copy_(torch.randn(p.shape, generator=gen) * (1.5 / max(p.shape[-1], 1) ** 0.5 if p.dim() > 1 else 0.3))
    m = m.to(DEV).eval()
    times = np.unique(quads[:, 3])
    g = torch.Generator().manual_seed(2)
    m.global_emb = {int(t): 0.1 * torch.randn(1, 1, H, generator=g) for t in times}
    m.graph_dict = synthetic.build_graph_dict(quads, NUM_R)
    S, ST, O, OT = synthetic.build_history(quads)
    t = quads[:, 3]
    tr, va, te = np.flatnonzero(t < 240), np.flatnonzero((t >= 240) & (t < 288)), np.flatnonzero(t >= 288)
    pick = lambda L, idx: [L[i] for i in idx]                                           # noqa: E731
    m.init_history(quads[tr], (pick(S, tr), pick(ST, tr)), (pick(O, tr), pick(OT, tr)),
                   quads[va], (pick(S, va), pick(ST, va)), (pick(O, va), pick(OT, va)),
                   quads[te], (pick(S, te), pick(ST, te)), (pick(O, te), pick(OT, te)))
    m.latest_time = torch.tensor(288)
    return m, StubGlobalModel(NUM_E, H, 17)


def _loop_roll_over(self, t, global_model):
    """The roll-over's candidate scoring as it was before pred_r_topk: pred_r_rank2 and torch.topk once per pick."""
    from collections import defaultdict

    from renet_b200.graph import get_big_graph
    from renet_b200.inference import history_triples
    K, R = self.num_k, self.num_rels
    last = {}
    for subject in (True, False):
        cache = self.s_his_cache if subject else self.o_his_cache
        cache_t = self.s_his_cache_t if subject else self.o_his_cache_t
        if subject:
            _, _, prob = global_model.predict(self.latest_time, self.graph_dict, subject=True)
        else:
            _, logits, _ = global_model.predict(t, self.graph_dict, subject=False)
            prob = torch.softmax(logits.view(-1), dim=0)
        picks = torch.distributions.categorical.Categorical(prob).sample(torch.Size([K]))
        lists, inds, ents = [], [], []
        for e, p_e in zip(picks, prob[picks]):
            ee = torch.full((R,), int(e), dtype=torch.long)
            joint = float(p_e) * self.pred_r_rank2(ee, torch.arange(R), subject=subject)
            top_p, top_i = torch.topk(joint.view(-1), K, sorted=False)
            lists.append(top_p.view(-1).cpu())
            inds.append(top_i.view(-1).cpu())
            ents.append(int(e))
        _, cand = torch.topk(torch.cat(lists), K, sorted=False)
        for c in cand.tolist():
            e = ents[c // K]
            last[subject] = e
            code = inds[c // K][c % K]
            rr, other = code // self.in_dim, code % self.in_dim
            cache[e] = self.update_cache(cache[e], rr, other.view(-1, 1))
            cache_t[e] = int(self.latest_time)
    self.data = history_triples(self.s_his_cache, self.o_his_cache)
    lt = int(self.latest_time)
    self.graph_dict[lt] = get_big_graph(self.data, R)
    self.global_emb[lt] = global_model.predict(self.latest_time, self.graph_dict, subject=True)[0]
    for hist, hist_t, cache, cache_t in ((self.s_hist_test, self.s_hist_test_t, self.s_his_cache, self.s_his_cache_t),
                                         (self.o_hist_test, self.o_hist_test_t, self.o_his_cache, self.o_his_cache_t)):
        for ee in range(self.in_dim):
            if len(cache[ee]) != 0:
                while len(hist[ee]) >= self.seq_len:
                    hist[ee].pop(0)
                    hist_t[ee].pop(0)
                hist[ee].append(torch.as_tensor(cache[ee]).cpu().numpy().copy())
                hist_t[ee].append(cache_t[ee])
                cache[ee] = []
                cache_t[ee] = None
    self.latest_time = t
    self.data = None
    self.preds_list_s = defaultdict(lambda: torch.zeros(self.num_k))
    self.preds_ind_s = defaultdict(lambda: torch.zeros(self.num_k))
    self.preds_list_o = defaultdict(lambda: torch.zeros(self.num_k))
    self.preds_ind_o = defaultdict(lambda: torch.zeros(self.num_k))
    return last[True], last[False]


def _state(m):
    from renet_b200.graph import as_history_graph
    graphs = {}
    for t, g in m.graph_dict.items():
        hg = as_history_graph(g)
        graphs[int(t)] = (hg.node_id.copy(), hg.src.copy(), hg.dst.copy(), hg.type_s.copy(), hg.type_o.copy())
    return dict(hist=[[np.asarray(a).tolist() for a in h] for h in m.s_hist_test + m.o_hist_test],
                hist_t=[list(map(int, h)) for h in m.s_hist_test_t + m.o_hist_test_t],
                cache=[np.asarray(c).tolist() for c in m.s_his_cache + m.o_his_cache],
                cache_t=list(m.s_his_cache_t) + list(m.o_his_cache_t), graphs=graphs,
                glob=sorted(int(t) for t in m.global_emb), latest=int(m.latest_time))


def _assert_same_state(a, b):
    for key in a:
        if key == 'graphs':
            assert sorted(a[key]) == sorted(b[key])
            for t in a[key]:
                for x, y in zip(a[key][t], b[key][t]):
                    np.testing.assert_array_equal(x, y)
        else:
            assert a[key] == b[key], key


def test_pred_r_topk_matches_per_entity_loop():
    quads = _stream()
    m, _ = _model(quads)
    R = NUM_R
    ents = [0, 5, 17, 5, 123, 299] + [int(e) for e in np.unique(quads[quads[:, 3] < 240][:, 0])[:20]]
    no_hist = [e for e in range(NUM_E) if len(m.s_hist_test[e]) == 0][:3]
    assert no_hist, 'the fixture needs entities without history'
    ents += no_hist
    gen = torch.Generator().manual_seed(9)
    wts = torch.rand(len(ents), generator=gen) * 0.1 + 1e-3
    with torch.no_grad():
        for subject in (True, False):
            vals, codes = m.pred_r_topk(ents, wts, NUM_K, subject=subject)
            for i, e in enumerate(ents):
                joint = float(wts[i]) * m.pred_r_rank2(torch.full((R,), e, dtype=torch.long), torch.arange(R), subject=subject)
                tp, ti = torch.topk(joint.view(-1), NUM_K, sorted=False)
                assert torch.equal(codes[i], ti), (subject, e)
                assert float(((vals[i] - tp).abs() / tp).max()) < 1e-5, (subject, e)


def test_rollover_matches_per_entity_loop():
    quads = _stream()
    m_new, gm_new = _model(quads)
    m_old, gm_old = _model(quads)
    _assert_same_state(_state(m_new), _state(m_old))
    picks_seen = []
    real_sampler = torch.distributions.categorical.Categorical.sample

    def spy(self, shape=torch.Size()):
        out = real_sampler(self, shape)
        picks_seen.append(out.clone())
        return out
    with torch.no_grad():
        for t_next in (312, 336):                        # two roll-overs: the second one sees the first's predicted graph
            torch.manual_seed(100 + t_next)
            torch.distributions.categorical.Categorical.sample = spy
            try:
                last_old = _loop_roll_over(m_old, torch.tensor(t_next), gm_old)
                rng_old = torch.get_rng_state()
                torch.manual_seed(100 + t_next)
                last_new = m_new._roll_over(torch.tensor(t_next), gm_new)
                rng_new = torch.get_rng_state()
            finally:
                torch.distributions.categorical.Categorical.sample = real_sampler
            assert last_new == last_old
            assert torch.equal(rng_new, rng_old)
            _assert_same_state(_state(m_new), _state(m_old))
    assert gm_new.calls == gm_old.calls
    # the fixture exercised repeated picks and picks without history
    for picks in picks_seen:
        assert len(torch.unique(picks)) < len(picks)
        assert bool((picks >= 250).any())
