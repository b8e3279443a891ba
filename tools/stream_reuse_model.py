"""How much of the stream gather's per-edge L2 traffic resident rows save, counted from the benchmark's own batches (CPU).

    python tools/stream_reuse_model.py [icews18|gdelt] [batches=1]

Replays bench.py's batches (the synthetic preset, seed 999, batch size 1024, both directions) through the host batcher
(utils.assemble_history_batch_host), cuts each graph into the kernel's 132 node-aligned CTA shares (a destination costs
2 edges; tests/test_stream_partition.py restates the rule) and counts, per CTA:
  * the reuse of source nodes: distinct sources / edges, the share of edges from the CTA's 32 / 64 most frequent sources,
    and the span of its source node ids (the hub histogram covers 2048 ids from the smallest);
  * the bytes its edge loop moves from L2 with H relation rows (the dataset ranking, GraphStore.hot_relations) and K hub
    source rows (the kernel's choice: the K most frequent of the 2048 ids from the CTA's smallest source, at least 2
    edges) resident: 800 B per edge whose source is not resident, 1600 B per edge whose relation is not.
Layer 1 is the batched history graph; layer 2 is its read-out sub-graph (renet_readout_subgraph restated: S compact
destinations, the distinct read-out nodes in ascending order, sources keep the full graph's ids).
These are counts from the data, not timings."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from renet_b200 import hoststore, synthetic, utils  # noqa: E402
from test_stream_partition import GRID, cta_boundary  # noqa: E402

BINS = 2048
CONFIGS = [(82, 0), (66, 32), (50, 64), (49, 64), (34, 96)]      # (H relation rows, K hub rows): about the same 131 KB


def hub_choice(srcs, k):
    """the kernel's hub choice for one CTA's source ids (StCfg HUB = k): set of ids"""
    if k == 0 or len(srcs) == 0:
        return set()
    lo = int(srcs.min())
    c = np.minimum(np.bincount(srcs[srcs < lo + BINS] - lo, minlength=BINS), 255)
    thr = next(t for t in range(2, 257) if (c >= t).sum() <= k)
    chosen = list(np.flatnonzero(c >= thr))
    if thr - 1 >= 2:
        chosen += list(np.flatnonzero(c == thr - 1)[:k - len(chosen)])
    return {lo + int(b) for b in chosen}


def shares(rp):
    N, E = len(rp) - 1, int(rp[-1])
    b = [cta_boundary(rp, N, E, c) for c in range(GRID + 1)]
    return [(b[c][1], b[c + 1][1]) for c in range(GRID)]


def model(rp, src, et, ranking, label):
    cut = [(cb, ce) for cb, ce in shares(rp) if ce > cb]
    stats = {'distinct/edges': [], 'top32': [], 'top64': [], 'span': []}
    for cb, ce in cut:
        s = src[cb:ce]
        cnt = np.sort(np.bincount(s - s.min()))[::-1]
        stats['distinct/edges'].append((cnt > 0).sum() / len(s))
        stats['top32'].append(cnt[:32].sum() / len(s))
        stats['top64'].append(cnt[:64].sum() / len(s))
        stats['span'].append(int(s.max() - s.min()) + 1)
    print('%s: %d destinations, %d edges, %d CTAs with edges' % (label, len(rp) - 1, int(rp[-1]), len(cut)))
    print('  per CTA (median): distinct sources / edges %.3f, edges from its 32 / 64 most frequent sources %.1f %% / %.1f %%,'
          ' source-id span %d (90th percentile %d, CTA 0 %d)' % (
              np.median(stats['distinct/edges']), 100 * np.median(stats['top32']), 100 * np.median(stats['top64']),
              np.median(stats['span']), np.percentile(stats['span'], 90), stats['span'][0]))
    E = int(rp[-1])
    for H, K in CONFIGS:
        hot = np.zeros(max(int(et.max()) + 1, len(ranking)), dtype=bool)
        hot[ranking[:H]] = True
        per_cta, hub_share = [], []
        for cb, ce in cut:
            s, t = src[cb:ce], et[cb:ce]
            res = np.isin(s, list(hub_choice(s, K))) if K else np.zeros(len(s), dtype=bool)
            per_cta.append(800 * int((~res).sum()) + 1600 * int((~hot[t]).sum()))
            hub_share.append(res.mean())
        print('  H %3d relation rows / K %3d hub rows (%.1f KB): %4.0f B per edge, busiest CTA %5.0f KB, edges from hubs %.1f %%'
              ' (median CTA), cold-relation edges %.1f %%' % (
                  H, K, (H * 1600 + K * 800) / 1000, sum(per_cta) / E, max(per_cta) / 1000, 100 * np.median(hub_share),
                  100 * (~hot[et[:E]]).mean()))


def readout_subgraph(rp, src, et, readout):
    uniq = np.unique(readout)
    deg = rp[uniq + 1] - rp[uniq]
    rp2 = np.concatenate(([0], np.cumsum(deg), np.full(len(readout) - len(uniq), deg.sum())))
    idx = np.concatenate([np.arange(rp[v], rp[v + 1]) for v in uniq]) if len(uniq) else np.zeros(0, np.int64)
    return rp2, src[idx], et[idx]


def main():
    preset = sys.argv[1] if len(sys.argv) > 1 else 'icews18'
    n_batches = int(([a[8:] for a in sys.argv[2:] if a.startswith('batches=')] or ['1'])[0])
    T = {'icews18': 240, 'gdelt': 2138}[preset]
    tkg = synthetic.SyntheticTKG(preset, seed=999, num_timestamps=T)
    gs = hoststore.GraphStore(tkg.graph_dict)
    for i in range(n_batches):
        q, sh, oh = tkg.batch(i, 1024, tail_only=False)
        for hist, col, reverse in ((sh, 0, False), (oh, 2, True)):
            hb = utils.assemble_history_batch_host(hist[0], hist[1], q[:, col], tkg.graph_dict)
            g = hb.graph
            rp, src = g['row_ptr'].astype(np.int64), g['col_src'].astype(np.int64)
            et = (g['col_type_o'] if reverse else g['col_type_s']).astype(np.int64)
            freq = np.bincount(gs.type_o if reverse else gs.type_s, minlength=gs.num_types)
            ranking = np.argsort(-freq, kind='stable')
            ranking = ranking[freq[ranking] > 0]
            side = 'object' if reverse else 'subject'
            model(rp, src, et, ranking, '%s batch %d, %s side, layer 1' % (preset, i, side))
            model(*readout_subgraph(rp, src, et, hb.readout_host), ranking, '%s batch %d, %s side, layer 2 (read-out sub-graph)'
                  % (preset, i, side))


if __name__ == '__main__':
    main()
