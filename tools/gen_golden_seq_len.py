"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/renet_seq_len.npz by running the UNMODIFIED reference at seq_len = 20,
as tools/gen_golden_relations.py writes its fixture (it needs the reference tree):

    python tools/gen_golden_seq_len.py

The stream: 16 entities, 4 relations, 30 timestamps; subjects are Zipf-distributed, so the hub entities take part in
nearly every timestamp and their histories reach 20 entries.  Stored, each at seq_len = 20:
  * RENet.forward (h = 8, 4 bases) on the 40 last quadruples, histories from build_history(history_len=20): the loss and
    every parameter gradient of both directions;
  * RENet_global.forward (h = 200, the reference's 100 bases) for a batch of timestamps whose windows hold 20 graphs, both
    poolings and directions: the loss and every gradient (the 600 x 200 GRU weights' as their norm and 1-D marginals);
    and get_global_emb over every timestamp (max pooling);
  * the test-time path (init_history, then evaluate_filter over the last two timestamps, with the stub global model of
    renet_eval_tiny): ranks, losses and scores per triple, and the test-time histories before and after the roll-over.
    The roll-over appends an entry to at least one history that already holds 20 entries, so the trim fires."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from oracle.gen_golden import OUT, RENET_SHAPES, det_global_emb, det_params  # noqa: E402

SEQ_LEN = 20


def stream():
    rng = np.random.RandomState(20)
    num_e, R, T = 16, 4, 30
    quads = []
    for t in range(T):
        n = rng.randint(24, 36)
        s = (rng.zipf(1.3, n) - 1) % num_e
        o = rng.randint(0, num_e, n)
        r = rng.randint(0, R, n)
        quads += [[a, b, c, t * 24] for a, b, c in zip(s, r, o)]
    return np.asarray(quads, dtype=np.int64), num_e, R


def store_grads(res, tag, model):
    """Every parameter gradient; a matrix of more than 20 000 elements as its norm and its two 1-D marginals, as
    oracle/gen_golden.run_renet stores them."""
    for k, p in model.named_parameters():
        if p.grad is None:
            continue
        if p.numel() > 20000 and p.dim() == 2:
            res['%s/grad_norm/%s' % (tag, k)] = np.float64(p.grad.double().norm().item())
            res['%s/grad_rowsum/%s' % (tag, k)] = p.grad.double().sum(1).numpy()
            res['%s/grad_colsum/%s' % (tag, k)] = p.grad.double().sum(0).numpy()
        else:
            res['%s/grad/%s' % (tag, k)] = p.grad.numpy().copy()


def renet_model(ns, num_e, R, h, nb, seed, num_k):
    m = ns.model.RENet(num_e, h, R, dropout=0, model=0, seq_len=SEQ_LEN, num_k=num_k)
    m.aggregator = ns.Aggregator.RGCNAggregator(h, 0, num_e, R, nb, 0, SEQ_LEN)
    m.load_state_dict(det_params(RENET_SHAPES(num_e, h, R, nb), seed), strict=True)
    return m


def gen(ns):
    from oracle import restate
    from oracle.stub_global import StubGlobalModel
    quads, num_e, R = stream()
    h, nb, seed = 8, 4, 31
    times = np.unique(quads[:, 3])
    S, ST, O, OT = restate.build_history(quads, num_e, history_len=SEQ_LEN)
    res = dict(quads=quads.astype(np.int32), num_e=num_e, R=R, h=h, nb=nb, seed=seed, seq_len=SEQ_LEN)
    with ref_loader.cpu_patches():
        gd = {int(t): ns.utils.get_big_graph(quads[quads[:, 3] == t][:, :3], R) for t in times}
        # ---- training forward / backward
        sel = np.arange(len(quads) - 40, len(quads))
        res['sel'] = sel
        res['sel_hist_len'] = np.asarray([len(S[i]) for i in sel])
        m = renet_model(ns, num_e, R, h, nb, seed, 10)
        m.global_emb = det_global_emb(times, h, seed + 1)
        batch = torch.from_numpy(quads[sel])
        sh = ([S[i] for i in sel], [ST[i] for i in sel])
        oh = ([O[i] for i in sel], [OT[i] for i in sel])
        for subj in (True, False):
            m.zero_grad()
            loss = m(batch, sh, oh, gd, subject=subj)
            loss.backward()
            tag = 'subj' if subj else 'obj'
            res[tag + '/loss'] = np.float64(loss.item())
            store_grads(res, tag, m)
        # ---- global model
        tps, tpo = ns.utils.get_true_distribution(quads, num_e)
        res['true_prob_s'], res['true_prob_o'] = tps, tpo
        gsel = np.asarray([29, 21, 25, 3, 27, 22])
        res['g_sel'] = gsel
        for pool in (1, 0):
            g = ns.global_model.RENet_global(num_e, 200, R, dropout=0, model=3, seq_len=SEQ_LEN, num_k=10, maxpool=pool)
            shapes = {k: tuple(v.shape) for k, v in g.state_dict().items()}
            g.load_state_dict(det_params(shapes, seed + 5), strict=True)
            for subj in (True, False):
                g.zero_grad()
                loss = g(torch.from_numpy(times[gsel]), torch.from_numpy(tps[gsel]), torch.from_numpy(tpo[gsel]), gd,
                         subject=subj)
                loss.backward()
                tag = 'pool%d/%s' % (pool, 'subj' if subj else 'obj')
                res[tag + '/loss'] = np.float64(loss.item())
                store_grads(res, tag, g)
            if pool == 1:
                with torch.no_grad():
                    ge = g.get_global_emb(times, gd)
                res['global_emb_keys'] = np.asarray(list(ge))
                res['global_emb'] = np.stack([ge[k].view(-1).numpy() for k in ge])
        # ---- test-time path
        t_valid, t_test = times[-4], times[-2]
        split = lambda lo, hi: np.flatnonzero((quads[:, 3] >= lo) & (quads[:, 3] < hi))   # noqa: E731
        tr, va, te = split(0, t_valid), split(t_valid, t_test), split(t_test, times[-1] + 1)
        pick = lambda L, idx: [L[i] for i in idx]                                           # noqa: E731
        num_k = 5
        m = renet_model(ns, num_e, R, h, nb, seed, num_k)
        m.eval()
        m.global_emb = det_global_emb(times, h, seed + 1)
        m.graph_dict = gd
        m.init_history(quads[tr], (pick(S, tr), pick(ST, tr)), (pick(O, tr), pick(OT, tr)),
                       quads[va], (pick(S, va), pick(ST, va)), (pick(O, va), pick(OT, va)),
                       quads[te], (pick(S, te), pick(ST, te)), (pick(O, te), pick(OT, te)))
        m.latest_time = torch.tensor(int(t_test))
        gm = StubGlobalModel(num_e, h, seed + 2)
        allq = torch.from_numpy(quads)
        torch.manual_seed(4321)
        out = {k: [] for k in ('filt', 'loss', 'sub_pred', 'ob_pred')}
        with torch.no_grad():
            for i in te:
                trip = torch.from_numpy(quads[i])
                if int(trip[3]) != int(m.latest_time):
                    res['before_len_s'] = np.array([len(x) for x in m.s_hist_test])
                    res['before_len_o'] = np.array([len(x) for x in m.o_hist_test])
                fr, loss = m.evaluate_filter(trip, (S[i], ST[i]), (O[i], OT[i]), gm, allq)
                if 'before_len_s' in res and 'rolled_at' not in res:
                    res['rolled_at'] = np.int64(i)
                    for side, hist_t in (('s', m.s_hist_test_t), ('o', m.o_hist_test_t)):
                        res['after_len_' + side] = np.array([len(x) for x in hist_t])
                        res['after_t_' + side] = np.array([list(x) + [-1] * (SEQ_LEN - len(x)) for x in hist_t])
                out['filt'].append(fr); out['loss'].append(loss.item())
                out['sub_pred'].append(m.predict(trip, (S[i], ST[i]), (O[i], OT[i]), gm)[1].numpy().copy())
                out['ob_pred'].append(m.predict(trip, (S[i], ST[i]), (O[i], OT[i]), gm)[2].numpy().copy())
    res.update({k: np.asarray(v) for k, v in out.items()})
    res.update(tr=tr, va=va, te=te, num_k=num_k, t_test=np.int64(t_test), gm_calls=np.asarray(gm.calls, dtype=np.int64))
    trimmed = sum(int(((res['before_len_' + x] == SEQ_LEN) & (res['after_t_' + x][:, -1] == t_test)).sum()) for x in 'so')
    assert trimmed > 0, 'the roll-over did not trim a full history'
    assert res['sel_hist_len'].max() == SEQ_LEN and (res['sel_hist_len'] > 16).sum() > 0
    np.savez_compressed(os.path.join(OUT, 'renet_seq_len.npz'), **res)
    print('renet_seq_len.npz: losses %.6f / %.6f, global %.6f, %d test triples, %d histories trimmed by the roll-over, '
          'batch history lengths %s' % (res['subj/loss'], res['obj/loss'], res['pool1/subj/loss'], len(te), trimmed,
                                        np.bincount(res['sel_hist_len']).tolist()))


if __name__ == '__main__':
    gen(ref_loader.load())
