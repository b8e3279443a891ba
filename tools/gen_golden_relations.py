"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/renet_relations_observed.npz by running the UNMODIFIED reference, as
tools/gen_golden_observed.py writes renet_eval_observed.npz (it needs the reference tree and tests/golden/renet_tiny.npz):

    python tools/gen_golden_relations.py

The relation head over observed history on the same tiny setup and the same triples (every triple of the last four
timestamps): per triple and direction, the reference's RGCNAggregator.predict over the triple's OWN ground-truth history
gives inp_r (Aggregator.py:218-237), ``encoder_r`` its final state s_q (zero for an empty history, model.py:187-189), and
``linear_r`` the logits of [ent_e | s_q] (model.py:202-208) -- the subject row over s's history (reverse=False), the object
row over o's object-side history (reverse=True, the inverse relation embeddings), as forward(subject=False) trains it.
Stored: the logits and their softmax; the rank of the triple's relation restated from the logits with the reference's tie
rule, raw (model.py:373-379) and filtered as evaluate_filter filters (model.py:391-405 applied to relations: the sigmoid,
every other relation r' of a known (s, r', .) -- or (., r', o) for the object row -- zeroed, the label kept), against all
quadruples and against those of the triple's own timestamp; and every row's full top-k (ids by softmax descending, ties
to the lower id, and their values)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from oracle.gen_golden import OUT, RENET_SHAPES, det_global_emb, det_params  # noqa: E402


def _rank(pred, label):
    """model.py:373-379 on one row."""
    comp1 = (pred > pred[label]).numpy()
    comp2 = (pred == pred[label]).numpy()
    return np.sum(comp1) + ((np.sum(comp2) - 1.0) / 2) + 1


def _filtered_rank(z, label, known_rels):
    """model.py:391-405 with relations as the answers: sigmoid, the known relations zeroed, the label kept."""
    pred = torch.sigmoid(z)
    ground = pred[label].clone()
    pred[known_rels] = 0
    pred[label] = ground
    return _rank(pred, label)


def gen_renet_relations_observed(ns):
    from oracle import restate
    blob = np.load(os.path.join(OUT, 'renet_tiny.npz'))
    quads = blob['quads'].astype(np.int64)
    num_e, R, h, nb, seed = int(blob['num_e']), int(blob['R']), int(blob['h']), int(blob['nb']), 21
    times = np.unique(quads[:, 3])
    rows = np.flatnonzero(quads[:, 3] >= times[-4])
    S, ST, O, OT = restate.build_history(quads, num_e)
    keys = ('z_s', 'z_o', 'p_s', 'p_o', 'raw', 'filt', 'time_filt', 'loss', 'topk_ids_s', 'topk_ids_o', 'topk_vals_s',
            'topk_vals_o')
    out = {k: [] for k in keys}
    with ref_loader.cpu_patches():
        gd = {int(t): ns.utils.get_big_graph(quads[quads[:, 3] == t][:, :3], R) for t in times}
        m = ns.model.RENet(num_e, h, R, dropout=0, model=0, seq_len=10, num_k=5)
        m.aggregator = ns.Aggregator.RGCNAggregator(h, 0, num_e, R, nb, 0, 10)
        m.load_state_dict(det_params(RENET_SHAPES(num_e, h, R, nb), seed), strict=True)
        m.eval()
        m.global_emb = det_global_emb(times, h, seed + 1)
        allq = torch.from_numpy(quads)

        def relation_logits(hist, hist_t, e, r, subject):
            if len(hist) == 0:
                s_q = torch.zeros(h)
            else:
                rel = m.rel_embeds[:R] if subject else m.rel_embeds[R:]
                _, inp_r = m.aggregator.predict((hist, hist_t), e, r, m.ent_embeds, rel, gd, m.global_emb,
                                                reverse=not subject)
                _, s_q = m.encoder_r(inp_r.view(1, len(hist), 3 * h))
                s_q = s_q.squeeze()
            return m.linear_r(torch.cat((m.ent_embeds[e], s_q), dim=0))

        with torch.no_grad():
            for i in rows:
                trip = torch.from_numpy(quads[i])
                s, r, o, t = trip[0], trip[1], trip[2], int(trip[3])
                z_s = relation_logits(S[i], ST[i], s, r, True)
                z_o = relation_logits(O[i], OT[i], o, r, False)
                lab = r.view(-1)
                out['loss'].append((m.criterion(z_s.view(1, -1), lab) + m.criterion(z_o.view(1, -1), lab)).item())
                raw, filt, tfilt = [], [], []
                for z, fix in ((z_s, 0), (z_o, 2)):
                    raw.append(_rank(z, int(r)))
                    for known, dst in ((allq, filt), (allq[allq[:, 3] == t], tfilt)):
                        dst.append(_filtered_rank(z, int(r), known[known[:, fix] == int(trip[fix])][:, 1]))
                out['raw'].append(raw); out['filt'].append(filt); out['time_filt'].append(tfilt)
                for z, side in ((z_s, 's'), (z_o, 'o')):
                    p = torch.softmax(z, dim=0)
                    order = torch.sort(p, descending=True, stable=True).indices
                    out['z_' + side].append(z.numpy().copy())
                    out['p_' + side].append(p.numpy().copy())
                    out['topk_ids_' + side].append(order.numpy().copy())
                    out['topk_vals_' + side].append(p[order].numpy().copy())
    res = {k: np.asarray(v) for k, v in out.items()}
    res.update(rows=rows, seed=seed,
               s_empty=np.asarray([len(S[i]) == 0 for i in rows]), o_empty=np.asarray([len(O[i]) == 0 for i in rows]))
    np.savez_compressed(os.path.join(OUT, 'renet_relations_observed.npz'), **res)
    print('renet_relations_observed.npz: %d triples, %d relations (%d / %d empty histories), mean raw / filtered / '
          'time-aware rank %.3f / %.3f / %.3f' % (len(rows), R, res['s_empty'].sum(), res['o_empty'].sum(), res['raw'].mean(),
                                                  res['filt'].mean(), res['time_filt'].mean()))


if __name__ == '__main__':
    gen_renet_relations_observed(ref_loader.load())
