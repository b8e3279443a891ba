"""Synthetic temporal knowledge graphs shaped like the reference's datasets, plus the DGL-free
preprocessing the hot path's inputs come from (reference data/<DS>/get_history_graph.py:137-190).

There is no network and the GPU box has no dataset files, so bench.py / smoke / the parity tests
drive the real batching pipeline with a synthetic quadruple stream whose statistics were fitted to
ICEWS18 (SURVEY.md Appendix A; measured from the reference's train.txt in the authoring container):
23,033 entities, 256 relations, ~1,554 events per timestamp, entity popularity ~ 1/(k+8)^1.2
(top-100 entities = 40 % of endpoints, top-1000 = 74 %), relation popularity with the top-10 = 63 %.
With batch 1024 over 240 timestamps this yields history graphs of ~239 components, ~34 k nodes, ~200 k directed
edges per direction (real ICEWS18, subject side: 32.9 k / 202 k; object side 41.9 k / 235 k) (see DESIGN.md for the side-by-side numbers).
"""
from collections import defaultdict

import numpy as np

from .graph import get_big_graph

PRESETS = {
    # name: (entities, relations, timestamps, events/timestamp, time step)
    'icews18': (23033, 256, 40, 1554, 24),
    'icews14': (12498, 260, 40, 1789, 24),
    'gdelt': (7691, 240, 60, 811, 15),
    'tiny': (60, 8, 14, 40, 24),
}


PAIR_FRACTION = 0.8
ENT_EXP, ENT_SHIFT, REL_EXP, REL_SHIFT = 1.2, 8.0, 1.25, 1.0
# per-preset (entity exponent, entity shift, pair fraction) where the ICEWS18 fit does not carry over.  GDELT (7,691
# entities, 2,138 timestamps of ~811 events over ~385 nodes each; batch of 1024: G ~ 2,083 components, N ~ 78 k,
# E ~ 462 k, SURVEY.md section 8(d) config 3): with these values and 2,138 timestamps the synthetic stream gives
# 405 nodes per timestamp and batches of G ~ 2,110, N ~ 72 k, E ~ 515 k.
SHAPE = {'gdelt': (1.2, 2.0, 1.0)}


def _power_law(n, a, q, rng):
    p = 1.0 / (np.arange(1, n + 1) + q) ** a
    p /= p.sum()
    return rng.permutation(n), p


def make_quads(preset='icews18', seed=999, num_timestamps=None):
    """int64 [n,4] (s, r, o, t), sorted by t like the reference's train.txt."""
    num_e, num_r, T, per_t, step = PRESETS[preset]
    T = num_timestamps or T
    rng = np.random.RandomState(seed)
    ent_exp, ent_shift, pair_fraction = SHAPE.get(preset, (ENT_EXP, ENT_SHIFT, PAIR_FRACTION))
    ent_perm, ent_p = _power_law(num_e, ent_exp, ent_shift, rng)
    rel_perm, rel_p = _power_law(num_r, REL_EXP, REL_SHIFT, rng)
    out = []
    for ti in range(T):
        n = max(4, int(rng.normal(per_t, per_t * 0.12)))
        # event = (pair, relation): a pool of distinct-ish entity pairs is drawn first and events re-use
        # pairs (the same two actors interact several times a day in ICEWS), which is what gives the
        # real graphs their multi-edges and ~6 mean in-degree
        n_pairs = max(2, int(n * pair_fraction))
        ps = ent_perm[rng.choice(num_e, n_pairs, p=ent_p)]
        po = ent_perm[rng.choice(num_e, n_pairs, p=ent_p)]
        clash = ps == po
        po[clash] = (po[clash] + 1) % num_e
        pick = rng.randint(0, n_pairs, n)
        s, o = ps[pick], po[pick]
        r = rel_perm[rng.choice(num_r, n, p=rel_p)]
        out.append(np.stack((s, r, o, np.full(n, ti * step)), axis=1))
    return np.concatenate(out).astype(np.int64), num_e, num_r


def build_graph_dict(quads, num_rels):
    """One graph per timestamp (get_history_graph.py:137-140)."""
    quads = np.asarray(quads, dtype=np.int64)
    order = np.argsort(quads[:, 3], kind='stable')
    q = quads[order]
    cuts = np.flatnonzero(np.diff(q[:, 3])) + 1
    out = {}
    for chunk in np.split(q, cuts):
        out[int(chunk[0, 3])] = get_big_graph(chunk[:, :3], num_rels)
    return out


def build_history(quads, history_len=10):
    """Rolling per-entity histories (get_history_graph.py:142-190): an entity's events of timestamp t
    become visible only once the stream moves past t; the last ``history_len`` timestamps are kept;
    each entry is an int array [k,2] of (relation, other entity) with its timestamp.
    Returns (s_hist, s_hist_t, o_hist, o_hist_t): one list per quadruple, as the reference pickles."""
    s_his, s_his_t = defaultdict(list), defaultdict(list)
    o_his, o_his_t = defaultdict(list), defaultdict(list)
    s_cache, o_cache = defaultdict(list), defaultdict(list)
    S, ST, O, OT = [], [], [], []
    latest_t = 0          # get_history_graph.py:131 (a first timestamp of 0 does not trigger a flush)

    def flush(cache, his, his_t, t_closed):
        for ee, ev in cache.items():
            if len(his[ee]) >= history_len:
                his[ee].pop(0)
                his_t[ee].pop(0)
            his[ee].append(np.asarray(ev, dtype=np.int64).reshape(-1, 2))
            his_t[ee].append(t_closed)
        cache.clear()

    for s, r, o, t in np.asarray(quads, dtype=np.int64).tolist():
        if latest_t != t:
            flush(s_cache, s_his, s_his_t, latest_t)
            flush(o_cache, o_his, o_his_t, latest_t)
            latest_t = t
        S.append(list(s_his[s])); ST.append(list(s_his_t[s]))
        O.append(list(o_his[o])); OT.append(list(o_his_t[o]))
        s_cache[s].append((r, o))
        o_cache[o].append((r, s))
    return S, ST, O, OT


def observed_history(facts, entities, timestamps, subject=True, history_len=10):
    """The history window of each (entities[i], timestamps[i]) over the known quadruples ``facts``: the reference's
    history of that entity at that time (get_history_graph.py:142-190), for any entity and time, not only those of a
    stream's quadruples.  It holds the last ``history_len`` distinct timestamps before t at which the entity is the subject
    of a fact (``subject=True``; its object otherwise), each entry an int64 array [k, 2] of (relation, other entity) in
    the facts' order.  Returns (lists, timestamp lists), one per query, as RENet.evaluate_observed and
    RENet.forecast_observed take them; for every quadruple of a time-sorted stream they equal build_history's.  The entry
    of one (entity, timestamp) is one array object, shared by every window that holds it, as in the reference's pickles.

    Vectorised: one stable sort of the facts by (entity, timestamp), whose runs are the entries, and one searchsorted per
    query for its window of runs; only the runs some window holds become arrays."""
    f = np.asarray(facts, dtype=np.int64)
    if f.ndim != 2 or f.shape[1] < 4:
        raise ValueError('observed_history: facts must be quadruples (s, r, o, t)')
    ents = np.asarray(entities, dtype=np.int64).reshape(-1)
    ts = np.asarray(timestamps, dtype=np.int64).reshape(-1)
    if len(ents) != len(ts):
        raise ValueError('observed_history: %d entities but %d timestamps' % (len(ents), len(ts)))
    if history_len < 1:
        raise ValueError('observed_history: history_len = %d, needs at least 1' % history_len)
    ent, other = (f[:, 0], f[:, 2]) if subject else (f[:, 2], f[:, 0])
    times, pos = np.unique(f[:, 3], return_inverse=True)
    T = len(times) + 1                                   # a query's position among the timestamps is at most len(times)
    key = ent * T + pos.reshape(-1)
    order = np.argsort(key, kind='stable')
    key = key[order]
    pairs = np.stack((f[order, 1], other[order]), axis=1)
    start = np.flatnonzero(np.concatenate(([True], key[1:] != key[:-1]))) if len(key) else np.zeros(0, np.int64)
    stop = np.append(start[1:], len(key))
    run_key = key[start]
    # the runs of entity e before t: keys in [e * T, e * T + #timestamps < t), the last history_len of them
    hi = np.searchsorted(run_key, ents * T + np.searchsorted(times, ts, 'left'), 'left')
    lo = np.maximum(np.searchsorted(run_key, ents * T, 'left'), hi - history_len)
    cover = np.zeros(len(start) + 1, dtype=np.int64)
    np.add.at(cover, lo, 1)
    np.add.at(cover, hi, -1)
    entry = [None] * len(start)
    for j in np.flatnonzero(np.cumsum(cover[:-1]) > 0).tolist():
        entry[j] = pairs[start[j]:stop[j]]
    run_t = times[run_key % T].tolist()
    lists = [entry[a:b] for a, b in zip(lo.tolist(), hi.tolist())]
    return lists, [run_t[a:b] for a, b in zip(lo.tolist(), hi.tolist())]


class SyntheticTKG:
    """quads + graph_dict + histories + a global_emb stand-in, ready for RENet.forward."""

    def __init__(self, preset='icews18', seed=999, num_timestamps=None, h_dim=200):
        import torch
        self.quads, self.num_e, self.num_r = make_quads(preset, seed, num_timestamps)
        self.graph_dict = build_graph_dict(self.quads, self.num_r)
        self.s_hist, self.s_hist_t, self.o_hist, self.o_hist_t = build_history(self.quads)
        g = torch.Generator().manual_seed(seed)
        # the reference's global_emb values are [1,1,h] tensors from the pre-trained global model
        self.global_emb = {t: 0.1 * torch.randn(1, 1, h_dim, generator=g) for t in self.graph_dict}

    def batch_indices(self, index, batch_size=1024, seed=999, tail_only=True):
        n = len(self.quads)
        lo = (2 * n) // 3 if tail_only else 0
        perm = np.random.RandomState(seed).permutation(np.arange(lo, n))
        return perm[(index * batch_size) % max(1, len(perm) - batch_size):][:batch_size]

    def batch(self, index, batch_size=1024, seed=999, tail_only=True):
        """``index``-th batch of a seeded permutation (train.py:127-129 shuffles then slices).  With
        tail_only the permutation covers the last third of the stream, where histories are full."""
        sel = self.batch_indices(index, batch_size, seed, tail_only)
        pick = lambda lst: [lst[i] for i in sel]
        return (self.quads[sel], (pick(self.s_hist), pick(self.s_hist_t)), (pick(self.o_hist), pick(self.o_hist_t)))
