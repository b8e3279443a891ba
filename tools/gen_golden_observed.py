"""TEST INFRASTRUCTURE ONLY -- writes tests/golden/renet_eval_observed.npz by running the UNMODIFIED reference, as
oracle/gen_golden.py writes the other fixtures (it needs the reference tree and tests/golden/renet_tiny.npz):

    python tools/gen_golden_observed.py

Evaluation over observed history on the tiny stream of renet_tiny.npz, for every triple of its last four timestamps: the
reference's RGCNAggregator.predict over the triple's OWN ground-truth history, then ``encoder`` (model.py:336-339 and
346-351 with (s_hist_i, s_hist_t_i) in place of s_hist_test[s]), zero rows for empty histories, and ``linear`` in both
directions, over the graphs and global embeddings of every timestamp.  The ranks come from the reference's own evaluate
(raw) and evaluate_filter (filtered against all quadruples, and time-aware: against the quadruples of the triple's own
timestamp), fed these scores through ``predict``.  Stored: scores, losses and the three rank sets."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from oracle.gen_golden import OUT, RENET_SHAPES, det_global_emb, det_params  # noqa: E402


def gen_renet_eval_observed(ns):
    from oracle import restate
    blob = np.load(os.path.join(OUT, 'renet_tiny.npz'))
    quads = blob['quads'].astype(np.int64)
    num_e, R, h, nb, seed = int(blob['num_e']), int(blob['R']), int(blob['h']), int(blob['nb']), 21
    times = np.unique(quads[:, 3])
    rows = np.flatnonzero(quads[:, 3] >= times[-4])
    S, ST, O, OT = restate.build_history(quads, num_e)
    out = {k: [] for k in ('raw', 'filt', 'time_filt', 'loss', 'sub_pred', 'ob_pred')}
    with ref_loader.cpu_patches():
        gd = {int(t): ns.utils.get_big_graph(quads[quads[:, 3] == t][:, :3], R) for t in times}
        m = ns.model.RENet(num_e, h, R, dropout=0, model=0, seq_len=10, num_k=5)
        m.aggregator = ns.Aggregator.RGCNAggregator(h, 0, num_e, R, nb, 0, 10)
        m.load_state_dict(det_params(RENET_SHAPES(num_e, h, R, nb), seed), strict=True)
        m.eval()
        m.global_emb = det_global_emb(times, h, seed + 1)
        allq = torch.from_numpy(quads)

        def encode(hist, hist_t, e, r, subject):
            if len(hist) == 0:
                return torch.zeros(h)
            rel = m.rel_embeds[:R] if subject else m.rel_embeds[R:]
            inp, _ = m.aggregator.predict((hist, hist_t), e, r, m.ent_embeds, rel, gd, m.global_emb, reverse=not subject)
            _, s_h = m.encoder(inp.view(1, len(hist), 4 * h))
            return s_h.squeeze()

        with torch.no_grad():
            for i in rows:
                trip = torch.from_numpy(quads[i])
                s, r, o = trip[0], trip[1], trip[2]
                s_h = encode(S[i], ST[i], s, r, True)
                o_h = encode(O[i], OT[i], o, r, False)
                ob_pred = m.linear(torch.cat((m.ent_embeds[s], s_h, m.rel_embeds[:R][r]), dim=0))
                sub_pred = m.linear(torch.cat((m.ent_embeds[o], o_h, m.rel_embeds[R:][r]), dim=0))
                loss = m.criterion(ob_pred.view(1, -1), o.view(-1)) + m.criterion(sub_pred.view(1, -1), s.view(-1))
                # the reference's own rank code, with these scores in place of its state's
                m.predict = lambda *a, **k: (loss, sub_pred.clone(), ob_pred.clone())   # noqa: E731
                raw, _ = m.evaluate(trip, None, None, None)
                filt, _ = m.evaluate_filter(trip, None, None, None, allq)
                tfilt, _ = m.evaluate_filter(trip, None, None, None, allq[allq[:, 3] == int(trip[3])])
                out['raw'].append(raw); out['filt'].append(filt); out['time_filt'].append(tfilt)
                out['loss'].append(loss.item())
                out['sub_pred'].append(sub_pred.numpy().copy()); out['ob_pred'].append(ob_pred.numpy().copy())
    res = {k: np.asarray(v) for k, v in out.items()}
    res.update(rows=rows, seed=seed,
               s_empty=np.asarray([len(S[i]) == 0 for i in rows]), o_empty=np.asarray([len(O[i]) == 0 for i in rows]))
    np.savez_compressed(os.path.join(OUT, 'renet_eval_observed.npz'), **res)
    print('renet_eval_observed.npz: %d triples (%d / %d empty histories), mean raw / filtered / time-aware rank %.3f / %.3f / '
          '%.3f' % (len(rows), res['s_empty'].sum(), res['o_empty'].sum(), res['raw'].mean(), res['filt'].mean(),
                    res['time_filt'].mean()))


if __name__ == '__main__':
    gen_renet_eval_observed(ref_loader.load())
