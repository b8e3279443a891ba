"""Test-time path of RE-Net on the H100 kernels (reference model.py:107-446; SURVEY.md section 8(f) row 2).

``RENetInference`` is mixed into ``renet_b200.model.RENet`` and provides the reference's evaluation API --
``init_history``, ``pred_r_rank2``, ``predict``, ``evaluate``, ``evaluate_filter``, ``update_cache`` -- with the same
arguments, return values and state attributes (``s_hist_test``, ``s_his_cache``, ``latest_time``, ``graph_dict``,
``global_emb`` ...), so the reference's ``test.py`` / validation loop (train.py:151-185) drive it unchanged.
``evaluate_filter_time`` and ``time_aware=True`` on ``evaluate_stream`` / ``evaluate_stream_batched`` add the time-aware
filter of the TKG forecasting literature: a query (s, r, ?, t) loses only the answers true at t.

Per-triple scoring runs history batching -> fused RGCN layers -> fused read-out + GRU through
``RGCNAggregator.encode`` (the same CUDA path as training); ranks use the reference's tie rule
``#greater + (#equal - 1) / 2 + 1`` (model.py:373-379).  The autoregressive roll-over on a timestamp change
(model.py:222-330) samples subjects/objects from the *global model*, which is outside this repo's scope: it is
passed in, as in the reference, and only needs ``predict(t, graph_dict, subject) -> (embedding, logits, prob)``.
"""
from collections import defaultdict

import numpy as np
import torch

from .graph import get_big_graph

#: (entity, relation) sequences pred_r_topk encodes and scores per chunk: 16 384 sequences of up to seq_len steps keep the
#: batched history graph, the GRU inputs and the decoder's partial sums within a few hundred MB
ROLLOVER_SEQ_BUDGET = 16384


def _seq_budget(max_len):
    """Sequences per encode chunk for histories of up to ``max_len`` steps: ROLLOVER_SEQ_BUDGET up to 16 steps, and
    16 / max_len of it above, so that the GRU's per-step buffers (8h floats per sequence and step) stay within their
    16-step size."""
    return ROLLOVER_SEQ_BUDGET if max_len <= 16 else max(1, ROLLOVER_SEQ_BUDGET * 16 // max_len)


#: distinct (entity, timestamp) components evaluate_stream_batched batches per chunk are bounded by their summed node and
#: candidate-edge counts: the plan's mark_off / cand_off are int32, and 2^28 keeps them far from overflow
EVAL_PLAN_BUDGET = 1 << 28


#: rows evaluate_observed ranks per renet_decoder_rank_multi call (two per triple): 16 384 rows of [ent | h | rel] at
#: h = 200 are 39 MB, and the call's per-row lists stay a few MB
OBSERVED_RANK_ROWS = 16384


def _isolated_view(hist, hist_t, subjects, samples, groups, graph_dict):
    """A HistoryView over a store of the histories hist / hist_t (one entry each, all non-empty, of subjects[i]) that
    selects ``samples`` (positions in hist), sample j in isolation group groups[j], over a GraphStore of the timestamps
    those histories reference.  Returns (view, graph store)."""
    from .hoststore import GraphStore, HistoryStore
    times = sorted({int(t) for ht in hist_t for t in ht})
    gs = GraphStore({t: graph_dict[t] for t in times})
    store = HistoryStore(list(hist), list(hist_t), np.asarray(subjects, dtype=np.int64), gs, dedupe=False)
    return store.select(np.asarray(samples, dtype=np.int64), groups=groups), gs


def _chunk_view(hist, hist_t, q_h, q_e, graph_dict):
    """The grouped view of one chunk of queries: query k has history hist[q_h[k]] / hist_t[q_h[k]] of entity q_e[k].  One
    store entry per distinct history, one isolation group per entity, so the batched graph's components are the distinct
    (entity, timestamp) pairs of the chunk.  Returns (view, graph store)."""
    uh, pos = np.unique(q_h, return_inverse=True)
    ue = np.zeros(len(uh), dtype=np.int64)
    ue[pos] = q_e
    group = np.unique(ue, return_inverse=True)[1].reshape(-1)
    return _isolated_view([hist[x] for x in uh], [hist_t[x] for x in uh], ue, pos.reshape(-1), group[pos.reshape(-1)],
                          graph_dict)


def rank_with_ties(scores, label):
    """model.py:373-379: rank = #(strictly greater) + (#equal - 1)/2 + 1."""
    ref = scores[label]
    greater = int((scores > ref).sum().item())
    equal = int((scores == ref).sum().item())
    return greater + (equal - 1.0) / 2 + 1


def history_triples(s_cache, o_cache):
    """utils.get_data (utils.py:95-113): the triples the per-entity caches describe.  A subject cache row (r, o) of
    entity i is (i, r, o); an object cache row (r, s) of entity i is (s, r, i); unique rows, sorted."""
    rows = []
    for i, c in enumerate(s_cache):
        if len(c) != 0:
            c = torch.as_tensor(c).cpu().long()
            rows.append(torch.cat((torch.full((len(c), 1), i, dtype=torch.long), c), dim=1))
    for i, c in enumerate(o_cache):
        if len(c) != 0:
            c = torch.as_tensor(c).cpu().long()
            rows.append(torch.stack((c[:, 1], c[:, 0], torch.full((len(c),), i, dtype=torch.long)), dim=1))
    if not rows:
        return None
    return np.unique(torch.cat(rows).numpy(), axis=0)


def stream_metrics(ranks, total_loss):
    """test.py:140-150: MRR / MR / Hits@{1,3,10} over all ranks, the summed loss and the ranks themselves."""
    ranks = np.concatenate(ranks) if ranks else np.zeros(0)
    out = {'mrr': float(np.mean(1.0 / ranks)) if len(ranks) else float('nan'),
           'mr': float(np.mean(ranks)) if len(ranks) else float('nan'), 'loss': total_loss, 'ranks': ranks}
    for k in (1, 3, 10):
        out['hits@%d' % k] = float(np.mean(ranks <= k)) if len(ranks) else float('nan')
    return out


#: the protocols evaluate_stream(time_aware=True) reports: raw (model.py:365-381), filtered by every answer known at any
#: time (model.py:384-419), and time-aware filtered by the answers known at the query's own timestamp only
PROTOCOLS = ('raw', 'filtered', 'time_filtered')


def _quadruples(total_data):
    """total_data as the time-aware filter needs it: known quadruples (s, r, o, t)."""
    if total_data is None:
        raise ValueError('time-aware evaluation needs total_data (all known quadruples)')
    q = torch.as_tensor(total_data)
    if q.dim() != 2 or q.shape[1] < 4:
        raise ValueError('time-aware evaluation needs total_data with a time column (s, r, o, t)')
    return q


def _same_time(all_triplets, triplet):
    """The rows of all_triplets at triplet's timestamp (column 3)."""
    allt = torch.as_tensor(all_triplets)
    return allt[allt[:, 3] == int(triplet[3])]


def _exclusion_lists(index, direction, *key):
    """(col, begin, end) of per-row exclusion lists from a FilterIndex / TimeFilterIndex: row i's list is the answers of
    key i ((fixed, r) or (fixed, r, t)) in direction 'subjects' where direction[i], else 'objects'; col holds both
    directions' columns."""
    b_ob, e_ob = index.ranges('objects', *key)
    b_sb, e_sb = index.ranges('subjects', *key)
    off = len(index.col('objects'))
    col = np.concatenate((index.col('objects'), index.col('subjects')))
    return col, np.where(direction, b_sb + off, b_ob), np.where(direction, e_sb + off, e_ob)


class FilterIndex:
    """The known answers of every (subject, relation) and (object, relation) pair of a set of triples, built once: what
    evaluate_filter (model.py:384-419) finds by scanning all triples for every test triple.  For direction ``objects``
    (the answers o of (s, r, ?)) and ``subjects`` (the answers s of (?, r, o)): one int32 column array of the sorted
    distinct answers, grouped by pair, and the pairs' keys sorted ascending."""

    def __init__(self, triples):
        t = np.asarray(torch.as_tensor(triples).cpu().numpy()[:, :3], dtype=np.int64)
        self.R = int(t[:, 1].max()) + 1 if len(t) else 1
        self.dirs = {}
        for name, fix, ans in (('objects', 0, 2), ('subjects', 2, 0)):
            u = np.unique(np.stack((t[:, fix] * self.R + t[:, 1], t[:, ans]), 1), axis=0) if len(t) else np.zeros((0, 2), np.int64)
            self.dirs[name] = (u[:, 0].copy(), np.ascontiguousarray(u[:, 1], dtype=np.int32))

    def ranges(self, direction, fixed, r):
        """(begin, end) int64 arrays: the answers of pair i are col(direction)[begin[i]:end[i]]."""
        keys, _ = self.dirs[direction]
        k = np.asarray(fixed, dtype=np.int64) * self.R + np.asarray(r, dtype=np.int64)
        k = np.where((np.asarray(r) >= 0) & (np.asarray(r) < self.R), k, -1)
        return np.searchsorted(keys, k, 'left'), np.searchsorted(keys, k, 'right')

    def col(self, direction):
        return self.dirs[direction][1]


class TimeFilterIndex:
    """FilterIndex keyed by (fixed entity, relation, timestamp), built once from quadruples: the answers the time-aware
    filter removes for a query (s, r, ?, t) or (?, r, o, t) -- those true at the query's own timestamp t only.  The same
    interface as FilterIndex, with the timestamp as one more key: ``ranges(direction, fixed, r, t)`` and
    ``col(direction)``.  Timestamps are replaced by their position among the distinct timestamps of the data, so the
    composite key (fixed * R + r) * T + position stays far inside int64 (1 M entities x 500 relations x T < 2^63 for any T up
    to 1.8e10)."""

    def __init__(self, quads):
        q = np.asarray(torch.as_tensor(quads).cpu().numpy(), dtype=np.int64)
        if q.ndim != 2 or q.shape[1] < 4:
            raise ValueError('TimeFilterIndex needs quadruples (s, r, o, t)')
        self.E = int(max(q[:, 0].max(), q[:, 2].max())) + 1 if len(q) else 1
        self.R = int(q[:, 1].max()) + 1 if len(q) else 1
        self.times = np.unique(q[:, 3])
        self.T = max(len(self.times), 1)
        if self.E * self.R * self.T >= 1 << 63:
            raise ValueError('TimeFilterIndex: %d entities x %d relations x %d timestamps overflow int64 keys'
                             % (self.E, self.R, self.T))
        pos = np.searchsorted(self.times, q[:, 3])
        self.dirs = {}
        for name, fix, ans in (('objects', 0, 2), ('subjects', 2, 0)):
            key = (q[:, fix] * self.R + q[:, 1]) * self.T + pos
            order = np.lexsort((q[:, ans], key))
            k, a = key[order], q[order, ans]
            keep = np.ones(len(k), dtype=bool)
            keep[1:] = (k[1:] != k[:-1]) | (a[1:] != a[:-1])           # distinct (key, answer) pairs
            self.dirs[name] = (k[keep], np.ascontiguousarray(a[keep], dtype=np.int32))

    def ranges(self, direction, fixed, r, t):
        """(begin, end) int64 arrays: the answers of query i are col(direction)[begin[i]:end[i]]; keys that are absent or
        out of range (entity, relation or timestamp) give empty ranges."""
        keys, _ = self.dirs[direction]
        fixed, r, t = (np.asarray(a, dtype=np.int64) for a in (fixed, r, t))
        fixed, r, t = np.broadcast_arrays(fixed, r, t)
        if len(self.times) == 0:
            z = np.zeros(fixed.shape, dtype=np.int64)
            return z, z
        pos = np.minimum(np.searchsorted(self.times, t), len(self.times) - 1)
        ok = (fixed >= 0) & (fixed < self.E) & (r >= 0) & (r < self.R) & (self.times[pos] == t)
        k = np.where(ok, (np.where(ok, fixed, 0) * self.R + np.where(ok, r, 0)) * self.T + pos, -1)
        return np.searchsorted(keys, k, 'left'), np.searchsorted(keys, k, 'right')

    def col(self, direction):
        return self.dirs[direction][1]


class RelationFilterIndex:
    """The known relations of every entity, built once from known facts: for an entity e as a subject, the r of every known
    (e, r, .); as an object, the r of every known (., r, e) -- the relations the filtered relation ranks leave out of a
    query (e, ?).  With ``time_aware=True`` (quadruples) keyed by (entity, timestamp): only the relations known at the
    query's own t.  Per side one int32 column array of the sorted distinct relations, grouped by key, and the keys sorted
    ascending; ``ranges(subject, entity[, t])`` and ``col(subject)`` give the CSR lists the rank and top-k kernels take."""

    def __init__(self, facts, time_aware=False):
        f = np.asarray(torch.as_tensor(facts).cpu().numpy(), dtype=np.int64)
        if f.ndim != 2 or f.shape[1] < (4 if time_aware else 3):
            raise ValueError('RelationFilterIndex needs %s' % ('quadruples (s, r, o, t)' if time_aware else 'triples (s, r, o)'))
        self.time_aware = time_aware
        self.times = np.unique(f[:, 3]) if time_aware else np.zeros(0, dtype=np.int64)
        self.T = max(len(self.times), 1)
        pos = np.searchsorted(self.times, f[:, 3]) if time_aware else 0
        self.sides = {}
        for subject, fix in ((True, 0), (False, 2)):
            key = f[:, fix] * self.T + pos
            order = np.lexsort((f[:, 1], key))
            k, r = key[order], f[order, 1]
            keep = np.ones(len(k), dtype=bool)
            keep[1:] = (k[1:] != k[:-1]) | (r[1:] != r[:-1])             # distinct (key, relation) pairs
            self.sides[subject] = (k[keep], np.ascontiguousarray(r[keep], dtype=np.int32))

    def ranges(self, subject, entity, t=None):
        """(begin, end) int64 arrays: the known relations of entity[i] (at t[i] when time-aware) on the given side are
        col(subject)[begin[i]:end[i]]; absent keys give empty ranges."""
        keys, _ = self.sides[bool(subject)]
        e = np.asarray(entity, dtype=np.int64)
        ok = e >= 0
        if self.time_aware:
            t = np.broadcast_to(np.asarray(t, dtype=np.int64), e.shape)
            if len(self.times) == 0:
                z = np.zeros(e.shape, dtype=np.int64)
                return z, z
            pos = np.minimum(np.searchsorted(self.times, t), len(self.times) - 1)
            ok &= self.times[pos] == t
            k = np.where(ok, np.where(ok, e, 0) * self.T + pos, -1)
        else:
            k = np.where(ok, e, -1)
        return np.searchsorted(keys, k, 'left'), np.searchsorted(keys, k, 'right')

    def col(self, subject):
        return self.sides[bool(subject)][1]


def _relation_exclusions(index, ents, subject, *t):
    """(col, begin, end) of per-row exclusion lists from a RelationFilterIndex: row i's list is the known relations of
    ents[i] (at t[i] when time-aware) on the subject side where subject[i], else on the object side; col holds both sides."""
    b_s, e_s = index.ranges(True, ents, *t)
    b_o, e_o = index.ranges(False, ents, *t)
    off = len(index.col(True))
    col = np.concatenate((index.col(True), index.col(False)))
    return col, np.where(subject, b_s, b_o + off), np.where(subject, e_s, e_o + off)


def rank_counts_torch(z, label, exclude=None):
    """What renet_decoder_rank counts, on materialised logits z [M, N] with torch: int64 [M, 4] = (#z > z_l, #z == z_l,
    #p > p_l, #p == p_l), p = torch.sigmoid(z) with row m's excluded columns other than its label set to 0 (the last two
    are 0 without ``exclude`` = (col, begin, end))."""
    M = z.shape[0]
    idx = torch.arange(M, device=z.device)
    zl = z[idx, label].view(-1, 1)
    out = torch.zeros(M, 4, dtype=torch.long, device=z.device)
    out[:, 0] = (z > zl).sum(1)
    out[:, 1] = (z == zl).sum(1)
    if exclude is not None:
        col, begin, end = (torch.as_tensor(x).long().cpu() for x in exclude)
        p = torch.sigmoid(z)
        for m in range(M):
            cols = col[begin[m]:end[m]].to(z.device)
            ground = p[m, label[m]].clone()
            p[m, cols] = 0
            p[m, label[m]] = ground
        pl = p[idx, label].view(-1, 1)
        out[:, 2] = (p > pl).sum(1)
        out[:, 3] = (p == pl).sum(1)
    return out


def topk_excluding_torch(z, k, exclude=None):
    """What renet_decoder_topk returns, on materialised logits z [M, N] with torch: per row the k largest p =
    softmax(z) over the columns outside row m's list col[begin[m]:end[m]] of ``exclude`` = (col, begin, end), by a stable
    descending sort (ties to the lower column; torch.topk leaves their order undefined); (values [M, k], indices int64
    [M, k]), index -1 and value 0 past a row's admissible columns."""
    p = torch.softmax(z, dim=1)
    key = p.clone()
    if exclude is not None:
        col, begin, end = (torch.as_tensor(a).long().cpu() for a in exclude)
        for m in range(len(z)):
            key[m, col[begin[m]:end[m]].to(z.device)] = -1.0         # below every probability
    order = torch.sort(key, dim=1, descending=True, stable=True).indices[:, :k]
    keep = torch.gather(key, 1, order) >= 0
    values = torch.where(keep, torch.gather(p, 1, order), torch.zeros((), dtype=p.dtype, device=p.device))
    return values, torch.where(keep, order, torch.full((), -1, dtype=torch.long, device=p.device))


class RENetInference:
    #: model.py:279,290 re-bind the local names ``s`` / ``o`` inside the roll-over loops, so the FIRST triple scored after
    #: every timestamp change is scored (and its loss taken) with the last subject / object candidate instead of its own
    #: (s, o).  True reproduces that (drop-in parity with the reference's numbers); False scores the triple itself.
    reference_rebinding = True

    # ---- state ----------------------------------------------------------------------------------------------------
    def init_history(self, triples, s_history, o_history, valid_triples, s_history_valid, o_history_valid,
                     test_triples=None, s_history_test=None, o_history_test=None):
        """model.py:107-166.  Per-entity test-time histories start from the training histories (last write wins), then
        take the validation / test ones whose newest entry is not newer than the last training timestamp."""
        n = self.in_dim
        self.s_hist_test = [[] for _ in range(n)]
        self.o_hist_test = [[] for _ in range(n)]
        self.s_hist_test_t = [[] for _ in range(n)]
        self.o_hist_test_t = [[] for _ in range(n)]
        self.s_his_cache = [[] for _ in range(n)]
        self.o_his_cache = [[] for _ in range(n)]
        self.s_his_cache_t = [None for _ in range(n)]
        self.o_his_cache_t = [None for _ in range(n)]
        last_t = None
        for tr, sh, sht, oh, oht in zip(triples, s_history[0], s_history[1], o_history[0], o_history[1]):
            s, o, last_t = int(tr[0]), int(tr[2]), tr[3]
            self.s_hist_test[s], self.s_hist_test_t[s] = list(sh), list(sht)
            self.o_hist_test[o], self.o_hist_test_t[o] = list(oh), list(oht)
        for trip, hs, ho in ((valid_triples, s_history_valid, o_history_valid), (test_triples, s_history_test, o_history_test)):
            if trip is None:
                continue
            for tr, sh, sht, oh, oht in zip(trip, hs[0], hs[1], ho[0], ho[1]):
                s, o = int(tr[0]), int(tr[2])
                if len(sht) != 0 and sht[-1] <= last_t:
                    self.s_hist_test[s], self.s_hist_test_t[s] = list(sh), list(sht)
                if len(oht) != 0 and oht[-1] <= last_t:
                    self.o_hist_test[o], self.o_hist_test_t[o] = list(oh), list(oht)

    def update_cache(self, cache, r, candidates):
        """model.py:421-446: add (r, candidate) rows to an entity's cache of predicted events, skipping candidates already
        present for relation r."""
        candidates = (candidates % self.in_dim).view(-1).long().cpu()
        r = torch.as_tensor(r).view(-1)[0].long().cpu()
        new = torch.stack((r.repeat(len(candidates)), candidates), dim=1)
        if len(cache) == 0:
            return new
        cache = torch.as_tensor(cache).cpu().long()
        known = cache[cache[:, 0] == r][:, 1]
        if len(known) != 0:
            keep = [i for i in range(len(candidates)) if candidates[i] not in known]
            if not keep:
                return cache
            new = new[torch.as_tensor(keep, dtype=torch.long)]
        return torch.cat((cache, new), dim=0)

    # ---- scoring ---------------------------------------------------------------------------------------------------------
    def _direction(self, subject):
        R = self.num_rels
        return (self.rel_embeds[:R], False) if subject else (self.rel_embeds[R:], True)

    def _encode_one(self, entity, r, history, history_t, subject, graph_dict=None, global_emb=None, relation=False):
        """Final hidden state of `encoder` for ONE (entity, relation) history (aggregator.predict + encoder,
        model.py:333-351), over the model's graph_dict / global_emb unless others are given.  ``relation=True``: the final
        state s_q of `encoder_r` instead (aggregator.predict's inp_r, model.py:94-96,200-204), which does not depend on r."""
        rel_embeds, reverse = self._direction(subject)
        dev = self.ent_embeds.device
        e = torch.as_tensor(entity, device=dev).view(1)
        rr = torch.as_tensor(r, device=dev).view(1)
        s_h, s_q, _ = self.aggregator.encode(([history], [history_t]), e, rr, self.ent_embeds, rel_embeds,
                                             self.graph_dict if graph_dict is None else graph_dict,
                                             self.global_emb if global_emb is None else global_emb, reverse, self.encoder,
                                             self.encoder_r)
        return (s_q if relation else s_h).view(-1)

    def pred_r_rank2(self, s, r, subject=True):
        """model.py:168-213: joint distribution over (relation, other entity) for entity s[0]:
        softmax_o(linear([ent[s], s_h(r), rel[r]])) * softmax_r(linear_r([ent[s], s_q]))."""
        R, h = self.num_rels, self.h_dim
        dev = self.ent_embeds.device
        ent = int(s[0])
        rel_embeds, reverse = self._direction(subject)
        hist = (self.s_hist_test if subject else self.o_hist_test)[ent]
        hist_t = (self.s_hist_test_t if subject else self.o_hist_test_t)[ent]
        s_dev = torch.as_tensor(s, device=dev).long().view(-1)
        r_dev = torch.as_tensor(r, device=dev).long().view(-1)
        if len(hist) == 0:
            s_h = torch.zeros(R, h, device=dev)
            s_q = torch.zeros(R, h, device=dev)
        else:
            # the same history for every relation (model.py:171-175): one component per timestamp, R read-out sequences
            s_h, s_q, _ = self.aggregator.encode(([hist] * R, [hist_t] * R), s_dev, r_dev, self.ent_embeds, rel_embeds,
                                                 self.graph_dict, self.global_emb, reverse, self.encoder, self.encoder_r)
        ob_pred = self.linear(torch.cat((self.ent_embeds[s_dev], s_h, rel_embeds), dim=1))
        p_o = torch.softmax(ob_pred.view(R, self.in_dim), dim=1)
        ob_pred_r = self.linear_r(torch.cat((self.ent_embeds[s_dev[0]], s_q[0]), dim=0))
        p_r = torch.softmax(ob_pred_r.view(-1), dim=0)
        return p_o * p_r.view(R, 1)

    def _grouped_view(self, entities, samples, subject):
        """A HistoryView over the current test-time histories of ``entities`` (all non-empty): one store entry per entity,
        the view's samples = ``samples`` (positions in ``entities``), each sample isolated in the group of its entity, over
        a GraphStore of the timestamps those histories reference.  Returns (view, graph store)."""
        hist = self.s_hist_test if subject else self.o_hist_test
        hist_t = self.s_hist_test_t if subject else self.o_hist_test_t
        samples = np.asarray(samples, dtype=np.int64)
        return _isolated_view([hist[e] for e in entities], [hist_t[e] for e in entities], entities, samples, samples,
                              self.graph_dict)

    def pred_r_topk(self, entities, weights, k, subject=True, capacity=None):
        """pred_r_rank2 followed by torch.topk for many entities at once (model.py:168-213, 236-240).  For entity
        entities[i]: the k largest entries of weights[i] * pred_r_rank2([entities[i]] * R, arange(R), subject).view(-1)
        and their codes r * in_dim + o, as (values float32 [n, k], codes int64 [n, k]) on the model's device.

        The test-time histories of a chunk of entities are encoded in one batched call (one store entry per entity, each
        repeated once per relation, through the C++ / device batcher with one isolation group per entity, so that every
        entity gets components of its own); entities without history get zero s_h / s_q as in
        pred_r_rank2.  The joint distribution is never materialised: renet_decoder_group_topk scores
        [ent_e | s_h(e, r) | rel_r] against ``linear`` with the row weights weights[i] * softmax_r(linear_r([ent_e | s_q_e]))
        and selects each entity's k best in one pass.  A group's k entries come in the order torch.topk(sorted=False) gives
        on a CUDA tensor of R * in_dim values (ORDER_INDEX: the values above the k-th one in index order, then those equal
        to it; measured on an H100 with PyTorch 2.11 from R * in_dim = 9 600 to 5.9 M), since the roll-over's final
        selection and the order of its cache updates depend on that layout."""
        ents, wts = self._topk_operands(entities, weights)
        n = len(ents)
        dev = self.ent_embeds.device
        values = torch.empty(n, k, device=dev)
        codes = torch.empty(n, k, dtype=torch.long, device=dev)
        for c0, c1 in self._topk_chunks(n):
            values[c0:c1], codes[c0:c1] = self._topk_chunk(ents[c0:c1], wts[c0:c1], k, subject, capacity)
        return values, codes

    def _topk_operands(self, entities, weights):
        """pred_r_topk's entities as a host int64 array and its weights as float32 on the model's device."""
        ents = torch.as_tensor(entities).reshape(-1).long().cpu().numpy()
        wts = torch.as_tensor(weights).reshape(-1).to(device=self.ent_embeds.device, dtype=torch.float32)
        if wts.numel() != len(ents):
            raise ValueError('pred_r_topk: %d entities but %d weights' % (len(ents), wts.numel()))
        return ents, wts

    def _topk_chunks(self, n):
        """[c0, c1) of pred_r_topk's chunks of n entities: _seq_budget(seq_len) // R entities each."""
        per = max(1, _seq_budget(self.seq_len) // self.num_rels)
        return [(c0, min(c0 + per, n)) for c0 in range(0, n, per)]

    def _topk_chunk(self, ce, wc, k, subject, capacity=None):
        """pred_r_topk of one chunk: host entities ``ce`` with device weights ``wc``, encoded and scored in one pass."""
        from .decoder import ORDER_INDEX, decoder_group_topk
        R, h = self.num_rels, self.h_dim
        dev = self.ent_embeds.device
        rel_embeds, reverse = self._direction(subject)
        hist = self.s_hist_test if subject else self.o_hist_test
        rel_rows = torch.arange(R, device=dev)
        nc = len(ce)
        s_h = torch.zeros(nc, R, h, device=dev)
        s_q = torch.zeros(nc, h, device=dev)
        has = np.flatnonzero([len(hist[e]) != 0 for e in ce])
        if len(has):
            he = ce[has]
            # The batched history graph has one component per timestamp, induced by the nodes of every sample in
            # the batch (utils.py:158-181), so an entity's encoding depends on what it is batched with.  One isolation
            # group per entity gives every entity components of its own, to encode exactly what pred_r_rank2 encodes
            # alone.
            view, gs = self._grouped_view(he, np.repeat(np.arange(len(he)), R), subject)
            s_dev = torch.from_numpy(np.repeat(he, R)).to(dev)
            r_dev = rel_rows.repeat(len(he))
            sh, sq, hb = self.aggregator.encode(view, s_dev, r_dev, self.ent_embeds, rel_embeds, gs, self.global_emb,
                                                reverse, self.encoder, self.encoder_r)
            # the encoder returns the sequences length-sorted: row j is sample sample_order[j] of the view
            idx = hb.sample_order(dev)
            sh_v, sq_v = torch.empty_like(sh), torch.empty_like(sq)
            sh_v[idx], sq_v[idx] = sh, sq
            has_dev = torch.from_numpy(has).to(dev)
            s_h[has_dev] = sh_v.view(len(he), R, h)
            s_q[has_dev] = sq_v.view(len(he), R, h)[:, 0]                 # s_q does not depend on r (model.py:96)
        ent = self.ent_embeds[torch.from_numpy(ce).to(dev)]
        p_r = torch.softmax(self.linear_r(torch.cat((ent, s_q), dim=1)), dim=1)                    # [nc, R]
        row_w = (wc.view(-1, 1) * p_r).reshape(-1)
        x = torch.cat((ent.repeat_interleave(R, dim=0), s_h.view(nc * R, h), rel_embeds.repeat(nc, 1)), dim=1)
        return decoder_group_topk(x, self.linear.weight, self.linear.bias, row_w, R, k, ORDER_INDEX, capacity)

    def _pick_candidates(self, draws, shard=None):
        """The num_k most probable (relation, entity) continuations of every pick (model.py:236-240), for each direction's
        draw (picks, prob, subject) of ``draws``: host tensors (joint probabilities [n_picks, num_k], codes r * in_dim + o
        [n_picks, num_k]) in picks order.  On the GPU every distinct entity of a draw is scored once, in pred_r_topk's
        chunks (its scores depend on the entity only), and its list is repeated for each pick of it.  A model on the host
        has no kernels to run (the host-logic checks substitute a host encoder): its picks are scored one by one through
        pred_r_rank2, as the reference does.

        The units of work -- the chunks of both directions on the GPU, the picks on the host -- are independent, and each
        gets exactly the operands it gets alone; with a ``shard`` (parallel.Shard) unit j runs on rank j mod world and
        every rank all-gathers the lists, so every rank returns what one process returns, bit for bit."""
        K, R = self.num_k, self.num_rels
        dev = self.ent_embeds.device
        jobs, done, inverse = [], [], []               # jobs: (draw, first row, end row) per unit, in unit order
        if self.ent_embeds.is_cuda:
            work = []
            for d, (picks, prob, subject) in enumerate(draws):
                uniq, inv = torch.unique(picks, return_inverse=True)
                work.append(self._topk_operands(uniq, prob[uniq]))
                inverse.append(inv.cpu())
                jobs += [(d, c0, c1) for c0, c1 in self._topk_chunks(len(uniq))]
            for j in (range(len(jobs)) if shard is None else shard.units(len(jobs))):
                d, c0, c1 = jobs[j]
                ents, wts = work[d]
                done.append(self._topk_chunk(ents[c0:c1], wts[c0:c1], K, draws[d][2]))
        else:
            jobs = [(d, i, i + 1) for d, (picks, _, _) in enumerate(draws) for i in range(len(picks))]
            inverse = [None] * len(draws)
            p_picks = [prob[picks] for picks, prob, _ in draws]          # each pick's probability
            for j in (range(len(jobs)) if shard is None else shard.units(len(jobs))):
                d, i, _ = jobs[j]
                picks, _, subject = draws[d]
                ee = torch.full((R,), int(picks[i]), dtype=torch.long)
                joint = float(p_picks[d][i]) * self.pred_r_rank2(ee, torch.arange(R), subject=subject)
                top_p, top_i = torch.topk(joint.view(-1), K, sorted=False)
                done.append((top_p.view(1, -1), top_i.view(1, -1)))
        vals, codes = [v for v, _ in done], [c for _, c in done]
        if shard is not None:
            sizes = [c1 - c0 for _, c0, c1 in jobs]
            vals = shard.gather_units(vals, sizes, torch.empty(0, K, device=dev))
            codes = shard.gather_units(codes, sizes, torch.empty(0, K, dtype=torch.long, device=dev))
        out = []
        for d in range(len(draws)):
            js = [j for j, job in enumerate(jobs) if job[0] == d]
            v, c = torch.cat([vals[j] for j in js]).cpu(), torch.cat([codes[j] for j in js]).cpu()
            out.append((v, c) if inverse[d] is None else (v[inverse[d]], c[inverse[d]]))
        return out

    def _roll_over(self, t, global_model, shard=None):
        """model.py:222-330: the stream moved to a new timestamp.  Sample num_k subjects (objects) from the global
        model's distribution, score every (relation, entity) continuation for them, keep the num_k most probable
        triples, turn them into the predicted graph of `latest_time`, and roll the per-entity histories.

        Both directions are sampled first, subject then object as the reference draws them: the global model reads
        graph_dict, which changes only after both directions, and the candidate scoring draws no random numbers, so the RNG
        stream and the global model's calls are the reference's.  Then both directions' candidates are scored together
        (_pick_candidates, sharded over ``shard`` when given) and the caches are updated in the reference's order."""
        K, R = self.num_k, self.num_rels
        draws = []
        for subject in (True, False):
            if subject:
                _, _, prob = global_model.predict(self.latest_time, self.graph_dict, subject=True)
            else:
                _, logits, _ = global_model.predict(t, self.graph_dict, subject=False)
                prob = torch.softmax(logits.view(-1), dim=0)                               # model.py:262
            picks = torch.distributions.categorical.Categorical(prob).sample(torch.Size([K]))
            draws.append((picks, prob, subject))
        if shard is not None:
            sums = [int((p.cpu().long() * torch.arange(1, len(p) + 1)).sum()) for p, _, _ in draws]
            if not shard.same_everywhere(sums):
                raise RuntimeError('evaluate_stream_batched: the ranks of process_group sampled different roll-over picks; '
                                   'they need the same torch seeds and a deterministic global model')
        last = {}
        # NOTE: the reference de-duplicates with a set of 0-dim tensors (model.py:228-234), which never matches (tensors
        # hash by identity), so repeated samples are scored again and kept as separate entries.
        for (picks, _, subject), (lists, inds) in zip(draws, self._pick_candidates(draws, shard)):   # [K picks, K] each
            cache = self.s_his_cache if subject else self.o_his_cache
            cache_t = self.s_his_cache_t if subject else self.o_his_cache_t
            ents = picks.tolist()
            _, cand = torch.topk(lists.view(-1), K, sorted=False)
            for c in cand.tolist():
                e = ents[c // K]
                last[subject] = e
                code = inds[c // K][c % K]
                rr, other = code // self.in_dim, code % self.in_dim
                cache[e] = self.update_cache(cache[e], rr, other.view(-1, 1))
                cache_t[e] = int(self.latest_time)
        self.data = history_triples(self.s_his_cache, self.o_his_cache)
        lt = int(self.latest_time)
        self.graph_dict[lt] = get_big_graph(self.data, R)                                # model.py:300-301
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

    def predict(self, triplet, s_hist, o_hist, global_model):
        """model.py:216-363 -> (loss, sub_pred [in_dim], ob_pred [in_dim])."""
        s, r, o = triplet[0], triplet[1], triplet[2]
        t = triplet[3].cpu()
        si, oi = int(s), int(o)
        if self.latest_time != t:
            last_s, last_o = self._roll_over(t, global_model)
            if self.reference_rebinding:
                si, oi = last_s, last_o
        R, h = self.num_rels, self.h_dim
        dev = self.ent_embeds.device
        if len(s_hist[0]) == 0 or len(self.s_hist_test[si]) == 0:
            s_h = torch.zeros(h, device=dev)
        else:
            s_h = self._encode_one(si, int(r), self.s_hist_test[si], self.s_hist_test_t[si], True)
        if len(o_hist[0]) == 0 or len(self.o_hist_test[oi]) == 0:
            o_h = torch.zeros(h, device=dev)
        else:
            o_h = self._encode_one(oi, int(r), self.o_hist_test[oi], self.o_hist_test_t[oi], False)
        ri = int(r)
        ob_pred = self.linear(torch.cat((self.ent_embeds[si], s_h, self.rel_embeds[:R][ri]), dim=0))
        sub_pred = self.linear(torch.cat((self.ent_embeds[oi], o_h, self.rel_embeds[R:][ri]), dim=0))
        o_lab = torch.as_tensor([oi], device=dev)
        s_lab = torch.as_tensor([si], device=dev)
        loss = self.criterion(ob_pred.view(1, -1), o_lab) + self.criterion(sub_pred.view(1, -1), s_lab)
        return loss, sub_pred, ob_pred

    def evaluate(self, triplet, s_hist, o_hist, global_model):
        """model.py:365-381: raw ranks (subject, object)."""
        loss, sub_pred, ob_pred = self.predict(triplet, s_hist, o_hist, global_model)
        return np.array([rank_with_ties(sub_pred, int(triplet[0])), rank_with_ties(ob_pred, int(triplet[2]))]), loss

    def evaluate_filter(self, triplet, s_hist, o_hist, global_model, all_triplets):
        """model.py:384-419: filtered ranks -- other known true answers of (s, r, ?) / (?, r, o) are zeroed after the
        sigmoid before ranking."""
        loss, sub_pred, ob_pred = self.predict(triplet, s_hist, o_hist, global_model)
        return self._filtered_ranks(triplet, sub_pred, ob_pred, all_triplets), loss

    def evaluate_filter_time(self, triplet, s_hist, o_hist, global_model, all_triplets):
        """evaluate_filter with the time-aware filter: only the answers known at the triple's own timestamp -- the rows of
        ``all_triplets`` whose column 3 equals triplet[3] -- are zeroed after the sigmoid.  Answers true at other times
        stay ranked, as a forecaster should rank them.  One predict call, as evaluate_filter."""
        loss, sub_pred, ob_pred = self.predict(triplet, s_hist, o_hist, global_model)
        return self._filtered_ranks(triplet, sub_pred, ob_pred, _same_time(all_triplets, triplet)), loss

    def _filtered_ranks(self, triplet, sub_pred, ob_pred, known):
        """evaluate_filter's ranking step (model.py:403-418) against the known triples ``known``: [subject, object] ranks."""
        s, r, o = int(triplet[0]), int(triplet[1]), int(triplet[2])
        sub_pred, ob_pred = torch.sigmoid(sub_pred), torch.sigmoid(ob_pred)
        allt = torch.as_tensor(known).to(ob_pred.device)
        ranks = []
        for pred, label, col_fix, col_out, fix in ((sub_pred, s, 2, 0, o), (ob_pred, o, 0, 2, s)):
            ground = pred[label].clone()
            ans = allt[(allt[:, col_fix] == fix) & (allt[:, 1] == r)][:, col_out].long()
            pred = pred.clone()
            pred[ans] = 0
            pred[label] = ground
            ranks.append(rank_with_ties(pred, label))
        return np.array(ranks)

    def evaluate_stream(self, test_data, s_history, o_history, global_model, total_data=None, raw=False, time_aware=False):
        """The reference's test loop (test.py:98-150) as a method: trims the per-entity histories to ``seq_len``
        (test.py:100-106), ranks every test triple in stream order (``evaluate`` when ``raw`` else ``evaluate_filter``
        against ``total_data``), and returns MRR / MR / Hits@{1,3,10} over subject and object ranks together, the summed
        loss and the ranks.  ``s_history`` / ``o_history`` = (lists, timestamp lists) of the test split.

        ``time_aware=True`` (``total_data`` = quadruples) scores each triple with one predict call and ranks its scores
        under all three protocols -- raw, filtered and time-aware filtered (evaluate_filter_time) -- returned as
        result['protocols'] = {'raw', 'filtered', 'time_filtered'}, each a dict like the result; the top-level keys stay
        the protocol ``raw`` selects.  (Calling evaluate, evaluate_filter and evaluate_filter_time in turn would run three
        predicts per triple, and the first triple after a roll-over is scored differently by the later ones.)"""
        self._trim_test_histories()
        test_data = torch.as_tensor(test_data)
        if time_aware:
            total_data = _quadruples(total_data)
        if not raw:
            if total_data is None:
                raise ValueError('filtered evaluation needs total_data (all known triples)')
        if not raw or time_aware:
            total_data = torch.as_tensor(total_data).to(self.ent_embeds.device)
        ranks, total_loss = [], 0.0
        protocols = {k: [] for k in PROTOCOLS}
        with torch.no_grad():
            for i in range(len(test_data)):
                trip = test_data[i].to(self.ent_embeds.device)
                sh, oh = (s_history[0][i], s_history[1][i]), (o_history[0][i], o_history[1][i])
                if time_aware:
                    loss, sub_pred, ob_pred = self.predict(trip, sh, oh, global_model)
                    protocols['raw'].append(np.array([rank_with_ties(sub_pred, int(trip[0])), rank_with_ties(ob_pred, int(trip[2]))]))
                    protocols['filtered'].append(self._filtered_ranks(trip, sub_pred, ob_pred, total_data))
                    protocols['time_filtered'].append(self._filtered_ranks(trip, sub_pred, ob_pred, _same_time(total_data, trip)))
                    r = protocols['raw' if raw else 'filtered'][-1]
                elif raw:
                    r, loss = self.evaluate(trip, sh, oh, global_model)
                else:
                    r, loss = self.evaluate_filter(trip, sh, oh, global_model, total_data)
                ranks.append(r)
                total_loss += float(loss)
        out = stream_metrics(ranks, total_loss)
        if time_aware:
            out['protocols'] = {k: stream_metrics(v, total_loss) for k, v in protocols.items()}
        return out

    def _trim_test_histories(self):
        """test.py:100-106: keep the last seq_len entries of every per-entity test-time history."""
        for hist, hist_t in ((self.s_hist_test, self.s_hist_test_t), (self.o_hist_test, self.o_hist_test_t)):
            for ee in range(self.in_dim):
                while len(hist[ee]) > self.seq_len:
                    hist[ee].pop(0)
                    hist_t[ee].pop(0)

    # ---- batched evaluation -------------------------------------------------------------------------------------------
    def evaluate_stream_batched(self, test_data, s_history, o_history, global_model, total_data=None, raw=False,
                                time_aware=False, process_group=None):
        """evaluate_stream, one timestamp at a time: same arguments, same result dict, same state afterwards (histories,
        caches, graph_dict, global_emb, latest_time, torch's RNG stream).  All triples of a timestamp are scored against the
        same state -- predict changes it only at the first triple of a new timestamp, through the roll-over -- so for each
        maximal run of equal timestamps the roll-over runs once, as predict runs it, and then every query of the run is
        encoded in one batched pass (one isolation group per entity, so each history is encoded as if alone) and every
        triple is scored and ranked by one renet_decoder_rank_multi call, with no exclusion list (``raw``) or one per row
        whose known answers come from a FilterIndex built once from ``total_data``.  A model on the host has no kernels: it
        encodes each query through _encode_one and ranks the materialised logits with torch, with the same grouping,
        rebinding and filter index.

        ``time_aware=True``: the call takes two lists per row, the static filter and the time-aware one (a TimeFilterIndex
        built once from the quadruples ``total_data``), and the result gets result['protocols'] as
        evaluate_stream(time_aware=True) returns it.

        ``process_group`` (a torch.distributed group, one process per GPU over NCCL, or gloo for a model on the host): every
        rank of the group calls with the same arguments, model state and torch seeds, and the work is sharded over the ranks
        in whole units of the one-process schedule -- the roll-over's candidate chunks (_pick_candidates), the query
        encoding chunks (_encode_queries) and contiguous row slices of each rank call (_score_run) -- each unit getting the
        operands it gets in one process.  Every rank then returns the result and ends in the state one process does, bit
        for bit; the host steps of the roll-over run on every rank.  None, or a group of one, runs unsharded.  Ranks called
        with different test data, latest_time, num_k or flags raise ValueError; ranks that sample different roll-over picks
        raise RuntimeError.  A caller outside the group raises ValueError.  A member of the group that never calls is not
        detected: the callers wait for it in the first all-gather, until the process group's own timeout (a collective
        cannot tell a late rank from an absent one)."""
        shard = self._eval_shard(process_group)
        test_data = torch.as_tensor(test_data)
        if shard is not None:
            self._check_ranks_agree(shard, test_data, len(s_history[0]), total_data, raw, time_aware)
        self._trim_test_histories()
        fidx = tfidx = None
        if time_aware:
            tfidx = TimeFilterIndex(_quadruples(total_data))
        if not raw or time_aware:
            if total_data is None:
                raise ValueError('filtered evaluation needs total_data (all known triples)')
            fidx = FilterIndex(total_data)
        protocols = {k: [] for k in PROTOCOLS}
        quads = test_data.cpu().numpy().astype(np.int64)
        s_empty = np.asarray([len(x) == 0 for x in s_history[0]], dtype=bool)
        o_empty = np.asarray([len(x) == 0 for x in o_history[0]], dtype=bool)
        ranks, total_loss = [], 0.0
        with torch.no_grad():
            i0, n = 0, len(quads)
            while i0 < n:
                i1 = i0 + 1
                while i1 < n and quads[i1, 3] == quads[i0, 3]:
                    i1 += 1
                t = test_data[i0][3].cpu()
                rebind = None
                if self.latest_time != t:                                   # predict's roll-over (model.py:222-330)
                    last_s, last_o = self._roll_over(t, global_model, shard)
                    if self.reference_rebinding:
                        rebind = (last_s, last_o)
                r, loss = self._score_run(quads[i0:i1], s_empty[i0:i1], o_empty[i0:i1], rebind, fidx, tfidx, shard)
                if time_aware:
                    for k in PROTOCOLS:
                        protocols[k].append(r[k])
                    r = r['raw' if raw else 'filtered']
                ranks.append(r)
                total_loss += float(np.sum(loss.astype(np.float64)))
                i0 = i1
        out = stream_metrics(ranks, total_loss)
        if time_aware:
            out['protocols'] = {k: stream_metrics(v, total_loss) for k, v in protocols.items()}
        return out

    def evaluate_observed(self, test_data, s_history, o_history, graph_dict, global_emb, total_data=None, raw=False,
                          time_aware=False):
        """Evaluation over observed history ("RE-Net w. GT"): every test triple (s, r, o, t) is encoded from its own
        ground-truth histories ``s_history`` / ``o_history`` = (lists, timestamp lists) per triple, as evaluate_stream takes
        them, over the true graphs ``graph_dict`` (e.g. synthetic.build_graph_dict of every known quadruple, a GraphStore,
        or the reference's dict) and the global embeddings ``global_emb`` of the timestamps those histories reference.
        Returns evaluate_stream_batched's result dict (``protocols`` with ``time_aware``, the top-level keys following
        ``raw``).

        Per triple: s_h = encoder(aggregator.predict(s's history, s, r)) (model.py:336-339 with the triple's own history in
        place of the test-time state), o_h the same on the object side (model.py:346-351), zero rows for empty histories;
        scores linear([ent | h | rel]) in both directions, ranked with the reference's tie rule raw, filtered
        (FilterIndex(total_data)) and time-aware filtered (TimeFilterIndex, keyed at the triple's own t); loss = predict's
        two cross-entropies.  Nothing rolls over and nothing is sampled: the test-time state (histories, caches,
        graph_dict, global_emb, latest_time) and torch's RNG are left as they are, so the call can run between
        evaluate_stream calls or inside a training loop.  The model scores in eval mode (no dropout) and its mode is
        restored.

        No timestamp depends on another, so the whole split is batched: each direction's distinct (entity, relation,
        history) queries are encoded once, in chunks through the device batcher with one isolation group per entity, whose
        components are the distinct (entity, history timestamp) pairs; then the rows are ranked OBSERVED_RANK_ROWS at a
        time by renet_decoder_rank_multi.  This needs the entries of one (entity, timestamp, direction) to be equal in every
        history that holds them, as histories built from one graph dict are; unequal ones raise ValueError, as do histories
        whose length differs from the test data's, ids out of range, history timestamps missing from graph_dict or
        global_emb, and ``time_aware`` without quadruples -- all before any work.  A model on the host takes the same flow
        through _encode_one and materialised logits."""
        quads, (s_obs, has_s), (o_obs, has_o) = self._observed_split(test_data, s_history, o_history, graph_dict, global_emb,
                                                                     total_data, raw, time_aware, 'evaluate_observed')
        n = len(quads)
        tfidx = TimeFilterIndex(_quadruples(total_data)) if time_aware else None
        fidx = FilterIndex(total_data) if not raw or time_aware else None
        protocols = {k: [] for k in PROTOCOLS}
        ranks, total_loss = [], 0.0
        modes = [(mod, mod.training) for mod in self.modules()]
        self.eval()
        try:
            with torch.no_grad():
                graphs = (graph_dict, global_emb)
                s_h = self._encode_queries(quads[:, 0], quads[:, 1], has_s, True, history=s_obs, graphs=graphs)
                o_h = self._encode_queries(quads[:, 2], quads[:, 1], has_o, False, history=o_obs, graphs=graphs)
                per = max(1, OBSERVED_RANK_ROWS // 2)
                for i0 in range(0, n, per):
                    i1 = min(i0 + per, n)
                    q = quads[i0:i1]
                    r, loss = self._rank_triples(q, q[:, 0], q[:, 2], s_h[i0:i1], o_h[i0:i1], fidx, tfidx)
                    if time_aware:
                        for k in PROTOCOLS:
                            protocols[k].append(r[k])
                        r = r['raw' if raw else 'filtered']
                    ranks.append(r)
                    total_loss += float(np.sum(loss.astype(np.float64)))
        finally:
            for mod, mode in modes:
                mod.training = mode
        out = stream_metrics(ranks, total_loss)
        if time_aware:
            out['protocols'] = {k: stream_metrics(v, total_loss) for k, v in protocols.items()}
        return out

    def _observed_split(self, test_data, s_history, o_history, graph_dict, global_emb, total_data, raw, time_aware, caller):
        """The checks of an observed-history evaluation, all before any work: (quads int64 [n, 4], (s_obs, has_s),
        (o_obs, has_o)) with each direction's histories as _observed_histories returns them.  ValueErrors name ``caller``."""
        test_data = torch.as_tensor(test_data)
        if test_data.dim() != 2 or test_data.shape[1] < 4:
            raise ValueError('%s: test_data must be quadruples (s, r, o, t)' % caller)
        quads = test_data.cpu().numpy().astype(np.int64)
        n = len(quads)
        if time_aware:
            _quadruples(total_data)
        if (not raw or time_aware) and total_data is None:
            raise ValueError('filtered evaluation needs total_data (all known triples)')
        for name, hist in (('s_history', s_history), ('o_history', o_history)):
            if len(hist) != 2 or len(hist[0]) != n or len(hist[1]) != n:
                raise ValueError('%s: %s must be (lists, timestamp lists) of %d test triples' % (caller, name, n))
        if n and (min(quads[:, 0].min(), quads[:, 2].min()) < 0 or max(quads[:, 0].max(), quads[:, 2].max()) >= self.in_dim):
            raise ValueError('%s: entity ids outside [0, %d)' % (caller, self.in_dim))
        if n and (quads[:, 1].min() < 0 or quads[:, 1].max() >= self.num_rels):
            raise ValueError('%s: relation ids outside [0, %d)' % (caller, self.num_rels))
        s = self._observed_histories(quads[:, 0], s_history, 's_history', graph_dict, global_emb, caller=caller)
        o = self._observed_histories(quads[:, 2], o_history, 'o_history', graph_dict, global_emb, caller=caller)
        return quads, s, o

    def evaluate_relations_observed(self, test_data, s_history, o_history, graph_dict, global_emb, total_data=None, raw=False,
                                    time_aware=False):
        """The relation head over observed history: how well p(r | s, history) -- what ``encoder_r`` + ``linear_r`` learn
        through training's 0.1-weighted relation loss (model.py:94-100) -- ranks the true relation of each test triple.
        Arguments, checks and result dict are evaluate_observed's.

        Per triple (s, r, o, t) two rows, each ranking the label r among all num_rels relations: the subject row
        linear_r([ent_s | s_q]), s_q the final state of ``encoder_r`` over s's own history (aggregator.predict's inp_r,
        reverse=False), and the object row linear_r([ent_o | o_q]) over o's object-side history (reverse=True), as
        forward(subject=False) trains it; an empty history gives a zero state (pred_r_rank2, model.py:187-189).  Ranks use
        the reference's tie rule: raw on the logits, filtered and time-aware filtered on the sigmoids with every other
        relation known for the row's entity on its side -- (s, r', .) for the subject row, (., r', o) for the object row --
        zeroed (RelationFilterIndex of ``total_data``, the time-aware one keyed at the row's own t).  ``ranks`` holds
        [subject row, object row] per triple and ``loss`` the sum of both rows' relation cross-entropies.

        Nothing rolls over, nothing is sampled and the global model is not called: the test-time state and torch's RNG are
        left as they are.  The model scores in eval mode and its mode is restored.  s_q does not depend on r, so each
        direction encodes each distinct (entity, history) once, through _encode_queries' chunks; the rows are ranked
        OBSERVED_RANK_ROWS at a time by renet_decoder_rank_multi against ``linear_r``.  A model on the host takes the same
        flow through _encode_one and materialised logits."""
        from .decoder import ranks_from_counts
        quads, (s_obs, has_s), (o_obs, has_o) = self._observed_split(test_data, s_history, o_history, graph_dict, global_emb,
                                                                     total_data, raw, time_aware,
                                                                     'evaluate_relations_observed')
        n = len(quads)
        indexes = []                                           # the static filter, then the time-aware one
        if not raw or time_aware:
            indexes.append(RelationFilterIndex(total_data))
        if time_aware:
            indexes.append(RelationFilterIndex(_quadruples(total_data), time_aware=True))
        dev = self.ent_embeds.device
        protocols = {k: [] for k in PROTOCOLS}
        ranks, total_loss = [], 0.0
        modes = [(mod, mod.training) for mod in self.modules()]
        self.eval()
        try:
            with torch.no_grad():
                graphs = (graph_dict, global_emb)
                s_q = self._encode_queries(quads[:, 0], None, has_s, True, history=s_obs, graphs=graphs,
                                           relation=True)
                o_q = self._encode_queries(quads[:, 2], None, has_o, False, history=o_obs, graphs=graphs,
                                           relation=True)
                per = max(1, OBSERVED_RANK_ROWS // 2)
                for i0 in range(0, n, per):
                    i1 = min(i0 + per, n)
                    q = quads[i0:i1]
                    m = i1 - i0
                    ents = np.concatenate((q[:, 0], q[:, 2]))
                    x = torch.cat((self.ent_embeds[torch.from_numpy(ents).to(dev)], torch.cat((s_q[i0:i1], o_q[i0:i1]))),
                                  dim=1)
                    side = np.concatenate((np.ones(m, bool), np.zeros(m, bool)))
                    t2 = np.concatenate((q[:, 3], q[:, 3]))
                    excludes = [_relation_exclusions(ix, ents, side, *((t2,) if ix.time_aware else ())) for ix in indexes]
                    loss_rows, counts = self._rank_rows(x, np.concatenate((q[:, 1], q[:, 1])), excludes, self.linear_r)
                    rks = [ranks_from_counts(counts[:, 2 * j], counts[:, 2 * j + 1]).cpu().numpy()
                           for j in range(len(excludes) + 1)]
                    pair = [np.stack((rk[:m], rk[m:]), axis=1).reshape(-1) for rk in rks]    # [subject, object] per triple
                    if time_aware:
                        for k, rk in zip(PROTOCOLS, pair):
                            protocols[k].append(rk)
                        ranks.append(pair[0] if raw else pair[1])
                    else:
                        ranks.append(pair[-1])
                    lr = loss_rows.cpu().numpy().astype(np.float32)
                    total_loss += float(np.sum((lr[:m] + lr[m:]).astype(np.float64)))
        finally:
            for mod, mode in modes:
                mod.training = mode
        out = stream_metrics(ranks, total_loss)
        if time_aware:
            out['protocols'] = {k: stream_metrics(v, total_loss) for k, v in protocols.items()}
        return out

    def _observed_histories(self, ents, history, name, graph_dict, global_emb, before=None, caller='evaluate_observed'):
        """evaluate_observed's histories of one direction, checked: ((hist, hist_t, hid, ent_of), has) -- the distinct
        histories (lists, timestamp lists), each triple's history id (-1 when empty), the entity of each history, and which
        triples have one.  A history is identified by its entity and timestamps, since the entries of one (entity, timestamp)
        must be equal wherever they appear (ValueError otherwise); ids ascend with the entity, as _encode_queries needs.
        ValueError for entry ids out of range, for timestamps missing from graph_dict or global_emb, and with ``before``
        (one timestamp per triple) for a history timestamp not before its triple's.  ValueErrors name ``caller``."""
        lists, times = history
        R, E = self.num_rels, self.in_dim
        seen = {}                                        # (entity, t) -> the first entry seen, as int64 [k, 2]
        keys = {}                                        # (entity, timestamps) -> first triple holding that history
        hid = np.full(len(ents), -1, dtype=np.int64)
        for i, (e, hl, ht) in enumerate(zip(ents.tolist(), lists, times)):
            if len(hl) != len(ht):
                raise ValueError('%s: %s[%d] has %d entries but %d timestamps' % (caller, name, i, len(hl), len(ht)))
            if len(hl) == 0:
                continue
            ts = tuple(int(t) for t in ht)
            if before is not None and max(ts) >= before[i]:
                # a forecast may only see the past: an entry at or after the query's timestamp may hold its answer
                raise ValueError('%s: %s[%d] holds timestamp %d, not before its query\'s timestamp %d'
                                 % (caller, name, i, max(ts), before[i]))
            for a, t in zip(hl, ts):
                prev = seen.get((e, t))
                if prev is None:
                    if t not in graph_dict:
                        raise ValueError('%s: %s[%d] refers to timestamp %d, which graph_dict lacks' % (caller, name, i, t))
                    if t not in global_emb:
                        raise ValueError('%s: %s[%d] refers to timestamp %d, which global_emb lacks' % (caller, name, i, t))
                    v = np.asarray(a, dtype=np.int64).reshape(-1, 2)
                    if len(v) and (v[:, 0].min() < 0 or v[:, 0].max() >= R or v[:, 1].min() < 0 or v[:, 1].max() >= E):
                        raise ValueError('%s: %s[%d] holds ids outside [0, %d) x [0, %d) at timestamp %d'
                                         % (caller, name, i, R, E, t))
                    seen[(e, t)] = (a, v)
                elif prev[0] is not a and not np.array_equal(prev[1], np.asarray(a, dtype=np.int64).reshape(-1, 2)):
                    raise ValueError('%s: %s[%d] holds an entry of entity %d at timestamp %d that differs from '
                                     'another history\'s entry of the same entity and timestamp' % (caller, name, i, e, t))
            hid[i] = keys.setdefault((e, ts), i)
        order = sorted(keys.items())                     # by entity, then timestamps
        rank = {first: j for j, (_, first) in enumerate(order)}
        has = hid >= 0
        hid[has] = [rank[x] for x in hid[has].tolist()]
        hist = [lists[first] for _, first in order]
        hist_t = [times[first] for _, first in order]
        ent_of = np.asarray([e for (e, _), _ in order], dtype=np.int64)
        return (hist, hist_t, hid, ent_of), has

    def _eval_shard(self, process_group, caller='evaluate_stream_batched'):
        """The parallel.Shard evaluate_stream_batched (or forecast, named by ``caller`` in errors) runs on, or None to run
        unsharded."""
        if process_group is None:
            return None
        import torch.distributed as dist
        from .parallel import Shard
        if not (dist.is_available() and dist.is_initialized()):
            raise ValueError('%s: process_group given, but torch.distributed is not initialised' % caller)
        if dist.get_rank(process_group) < 0:
            raise ValueError('%s: this process is not a member of process_group' % caller)
        if dist.get_world_size(process_group) == 1:
            return None
        if dist.get_backend(process_group) == 'nccl' and not self.ent_embeds.is_cuda:
            raise ValueError('%s: an NCCL process_group needs the model on a GPU; a model on the host takes a gloo group'
                             % caller)
        return Shard(process_group, self.ent_embeds.device)

    def _check_ranks_agree(self, shard, test_data, n_hist, total_data, raw, time_aware):
        """ValueError on every rank unless every rank of ``shard`` was called with the same test data (length and a hash of
        the quadruples), latest_time, num_k and flags: one small all-gather, before any work."""
        import hashlib
        q = np.ascontiguousarray(test_data.cpu().numpy().astype(np.int64))
        digest = int.from_bytes(hashlib.blake2b(q.tobytes(), digest_size=7).digest(), 'little')
        fp = [len(q), digest, int(self.latest_time), int(self.num_k), n_hist, int(total_data is None), int(bool(raw)),
              int(bool(time_aware)), int(bool(self.reference_rebinding))]
        if not shard.same_everywhere(fp):
            raise ValueError('evaluate_stream_batched: the ranks of process_group were called with different test data, '
                             'latest_time, num_k or flags')

    def _score_run(self, quads, s_empty, o_empty, rebind, fidx, tfidx=None, shard=None):
        """Scores the triples of one timestamp against the current state: (ranks float64 [2n] as [sub, ob] per triple,
        loss float32 [n] = predict's two cross-entropies per triple).  rebind = (s, o) of the roll-over that the run's first
        triple is scored with (model.py:279,290) or None; its rank labels and filter keys stay its own.  With a
        TimeFilterIndex ``tfidx`` (and ``fidx``) the ranks are a dict of the three PROTOCOLS, the time-aware keys taking the
        run's timestamp.  With a ``shard`` the encoding and the rank call are sharded over its ranks."""
        s, r, o = quads[:, 0].copy(), quads[:, 1].copy(), quads[:, 2].copy()
        si, oi = s.copy(), o.copy()
        if rebind is not None:
            si[0], oi[0] = rebind
        has_s = ~s_empty & np.asarray([len(self.s_hist_test[e]) != 0 for e in si], dtype=bool)
        has_o = ~o_empty & np.asarray([len(self.o_hist_test[e]) != 0 for e in oi], dtype=bool)
        s_h = self._encode_queries(si, r, has_s, True, shard)
        o_h = self._encode_queries(oi, r, has_o, False, shard)
        return self._rank_triples(quads, si, oi, s_h, o_h, fidx, tfidx, shard)

    def _rank_triples(self, quads, si, oi, s_h, o_h, fidx, tfidx=None, shard=None):
        """Scores and ranks the triples ``quads`` (s, r, o, t) given their encodings: the object of triple i against
        [ent[si[i]] | s_h[i] | rel[r]] and its subject against [ent[oi[i]] | o_h[i] | rel_inv[r]].  si / oi equal s / o
        except at row 0 of a rebound run (_score_run).  Returns (ranks float64 [2n] as [sub, ob] per triple, loss float32 [n]
        = predict's two cross-entropies per triple); with a TimeFilterIndex ``tfidx`` (and ``fidx``) the ranks are a dict
        of the three PROTOCOLS, the time-aware key of each row taking its own triple's timestamp.  With a ``shard`` the rank
        call is sharded over its ranks."""
        from .decoder import ranks_from_counts
        R = self.num_rels
        dev = self.ent_embeds.device
        n = len(quads)
        s, r, o, t = (np.ascontiguousarray(quads[:, j]) for j in range(4))
        to_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to(dev)    # noqa: E731
        si_d, oi_d, r_d = to_dev(si), to_dev(oi), to_dev(r)
        x = torch.cat((torch.cat((self.ent_embeds[si_d], s_h, self.rel_embeds[:R][r_d]), dim=1),
                       torch.cat((self.ent_embeds[oi_d], o_h, self.rel_embeds[R:][r_d]), dim=1)), dim=0)
        rank_lab = np.concatenate((o, s))                        # ob rows rank the triple's object, sub rows its subject
        loss_row = np.concatenate((np.arange(n), n + np.arange(n)))
        if n and (si[0] != s[0] or oi[0] != o[0]):
            # predict's loss for the rebound triple takes the rebound labels: two extra rows carry them
            x = torch.cat((x, x[[0, n]]), dim=0)
            rank_lab = np.concatenate((rank_lab, [oi[0], si[0]]))
            loss_row[0], loss_row[n] = 2 * n, 2 * n + 1
        # Each row's loss and counts depend on that row alone (the rank passes have no split-K and no kernel choice by row
        # count), so a shard ranks a contiguous slice of the rows, with the exclusion lists of its rows only.
        m = len(rank_lab)
        lo, hi = (0, m) if shard is None else shard.slice(m)
        excludes = []                                            # the static filter, then the time-aware one
        if fidx is not None:
            fix = np.concatenate((s, o, [s[0], o[0]]))[:m][lo:hi]
            rr = np.concatenate((r, r, [r[0], r[0]]))[:m][lo:hi]
            direction = np.concatenate((np.zeros(n, bool), np.ones(n, bool), [False, True]))[:m][lo:hi]
            excludes.append(_exclusion_lists(fidx, direction, fix, rr))
            if tfidx is not None:
                tt = np.concatenate((t, t, t[:1], t[:1]))[:m][lo:hi]
                excludes.append(_exclusion_lists(tfidx, direction, fix, rr, tt))
        loss_rows, counts = self._rank_rows(x[lo:hi], rank_lab[lo:hi], excludes)
        if shard is not None:
            loss_rows, counts = shard.allgather_slices(loss_rows, m), shard.allgather_slices(counts, m)
        rks = [ranks_from_counts(counts[:, 2 * j], counts[:, 2 * j + 1]) for j in range(len(excludes) + 1)]
        pair = lambda rk: np.stack((rk[n:2 * n], rk[:n]), axis=1).reshape(-1)    # noqa: E731
        if tfidx is None:
            ranks = pair(rks[-1].cpu().numpy())                  # filtered with a filter index, else raw
        else:
            ranks = {k: pair(rk.cpu().numpy()) for k, rk in zip(PROTOCOLS, rks)}
        lr = loss_rows.cpu().numpy().astype(np.float32)
        return ranks, lr[loss_row[:n]] + lr[loss_row[n:]]

    def _rank_rows(self, x, label, excludes, linear=None):
        """(loss_rows [M], counts [M, 2 + 2L]) of the rows of x against ``linear`` (the entity head's unless another is
        given): the raw (greater, equal) pair, then the filtered pair against each of the L = 0-2 exclusion lists
        ``excludes``.  One renet_decoder_rank_multi call on the GPU; on the host, row by row through ``linear`` as predict
        computes them, counted with torch once per list."""
        from .decoder import decoder_rank_counts_multi
        linear = self.linear if linear is None else linear
        dev = x.device
        lab = torch.from_numpy(np.ascontiguousarray(label, dtype=np.int64)).to(dev)
        if len(lab) == 0:
            # a shard without rows (fewer rows than ranks): nothing to launch, and the empty results keep the dtypes of
            # the other ranks' shares, which the all-gather after this call needs
            return (torch.zeros(0, device=dev),
                    torch.zeros(0, 2 + 2 * len(excludes), dtype=torch.int32 if x.is_cuda else torch.long, device=dev))
        if x.is_cuda:
            ex = [tuple(torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(dev) for a in e) for e in excludes]
            return decoder_rank_counts_multi(x, linear.weight, linear.bias, lab, ex)
        z = torch.stack([linear(row) for row in x])
        loss_rows = torch.stack([self.criterion(z[m].view(1, -1), lab[m].view(1)) for m in range(len(lab))])
        cs = [rank_counts_torch(z, lab, e) for e in excludes]
        return loss_rows, torch.cat([rank_counts_torch(z, lab)[:, :2]] + [ci[:, 2:] for ci in cs], dim=1)

    def _encode_queries(self, ents, rels, has, subject, shard=None, history=None, graphs=None, relation=False):
        """s_h [n, h] of the queries (ents[i], rels[i]); rows where ``has`` is False stay zero (predict's empty-history
        rule).  Query i's history is the current test-time history of ents[i], or with ``history`` = (hist, hist_t, hid,
        ent_of) the history hist[hid[i]] / hist_t[hid[i]], whose entity is ent_of[hid[i]] (= ents[i]), over ``graphs`` =
        (graph_dict, global_emb) instead of the model's.  Equal queries (history, relation) are encoded once.  On the GPU the
        distinct queries go through the device batcher in chunks, one isolation group per entity, so that each equals
        _encode_one's encoding of it alone; on the host, through _encode_one, one query per chunk.  With a ``shard`` chunk j
        runs on rank j mod world and every rank all-gathers the encodings.

        ``relation=True``: the relation head's s_q [n, h] instead, the final state of ``encoder_r`` that the same fused pass
        computes.  s_q does not depend on the relation (its inputs are [H2 | ent | global], model.py:94-96), so ``rels`` is
        ignored and each distinct history is encoded once."""
        h, R = self.h_dim, self.num_rels
        dev = self.ent_embeds.device
        out = torch.zeros(len(ents), h, device=dev)
        sel = np.flatnonzero(has)
        if len(sel) == 0:
            return out
        if relation:
            rels = np.zeros(len(ents), dtype=np.int64)
        graph_dict, global_emb = (self.graph_dict, self.global_emb) if graphs is None else graphs
        if history is None:
            hist = self.s_hist_test if subject else self.o_hist_test
            hist_t = self.s_hist_test_t if subject else self.o_hist_test_t
            hid, ent_of = np.asarray(ents), None
        else:
            hist, hist_t, hid, ent_of = history
        keys, inverse = np.unique(np.asarray(hid)[sel].astype(np.int64) * R + np.asarray(rels)[sel], return_inverse=True)
        q_h, q_r = keys // R, keys % R                   # history ids ascend with their entity, so keys are sorted by entity
        q_e = q_h if ent_of is None else np.asarray(ent_of, dtype=np.int64)[q_h]
        if not self.ent_embeds.is_cuda:
            chunks = [(j, j + 1) for j in range(len(keys))]
        else:
            rel_embeds, reverse = self._direction(subject)
            ent_times = defaultdict(set)                 # the timestamps of every history of each entity
            for hh, e in zip(*np.unique(np.stack((q_h, q_e), 1), axis=0).T):
                ent_times[e].update(int(t) for t in hist_t[hh])
            sizes = {}
            for t in set().union(*ent_times.values()):
                g = graph_dict[t]
                sizes[t] = g.number_of_nodes() + g.number_of_edges()
            budget = _seq_budget(max(self.seq_len, max(len(hist_t[hh]) for hh in np.unique(q_h))))
            chunks, j0 = [], 0
            while j0 < len(keys):
                # a chunk: whole entities, within both budgets; an entity's components are the distinct timestamps of its
                # histories
                cost, j1 = 0, j0
                while j1 < len(keys) and j1 - j0 < budget:
                    e = q_e[j1]
                    if j1 == j0 or e != q_e[j1 - 1]:
                        c = sum(sizes[t] for t in ent_times[e])
                        if j1 > j0 and cost + c > EVAL_PLAN_BUDGET:
                            break
                        cost += c
                    j1 += 1
                chunks.append((j0, j1))
                j0 = j1
        parts = []
        for j0, j1 in (chunks[c] for c in (range(len(chunks)) if shard is None else shard.units(len(chunks)))):
            if not self.ent_embeds.is_cuda:
                hh, e, rr = int(q_h[j0]), int(q_e[j0]), int(q_r[j0])
                parts.append(self._encode_one(e, rr, hist[hh], hist_t[hh], subject, graph_dict, global_emb, relation)
                             .view(1, h).to(out.dtype))
                continue
            view, gs = _chunk_view(hist, hist_t, q_h[j0:j1], q_e[j0:j1], graph_dict)
            s_dev = torch.from_numpy(q_e[j0:j1]).to(dev)
            r_dev = torch.from_numpy(q_r[j0:j1]).to(dev)
            sh, sq, hb = self.aggregator.encode(view, s_dev, r_dev, self.ent_embeds, rel_embeds, gs, global_emb,
                                                reverse, self.encoder, self.encoder_r)
            state = sq if relation else sh
            # the encoder returns the sequences length-sorted: row k is sample sample_order[k] of the view
            idx = hb.sample_order(dev)
            part = torch.empty_like(state)
            part[idx] = state
            parts.append(part)
        if shard is not None:
            parts = shard.gather_units(parts, [j1 - j0 for j0, j1 in chunks], out[:0])
        enc = torch.cat(parts)
        out[torch.from_numpy(sel).to(dev)] = enc[torch.from_numpy(inverse.reshape(-1)).to(dev)]
        return out

    # ---- forecasting ------------------------------------------------------------------------------------------------
    def forecast(self, queries, global_model, k=10, subject=True, known=None, time_aware=False, process_group=None):
        """The model's k most likely answers of each query, over its own test-time state as predict keeps it.

        ``queries``: int64 [n, 3] rows (entity, relation, timestamp), timestamps non-decreasing and not before
        ``latest_time``.  ``subject=True`` asks for the objects of (e, r, ?, t): the rows [ent_e | s_h(e, r) | rel_r]
        predict builds for its object scores; ``False`` for the subjects of (?, r, e, t), from the object-side history and
        the inverse relation embeddings.  Returns (values float32 [n, k], entity ids int64 [n, k]) on the model's device,
        values p = softmax over all entities, descending, ties to the lower id.

        For each run of equal timestamps the stream rolls over as evaluate_stream_batched rolls it (the same _roll_over: the
        same histories, caches, graph_dict, global_emb, latest_time and torch RNG stream afterwards), then the run's
        queries are encoded in one batched pass and scored by one renet_decoder_topk call.  Each query is scored as itself
        (``reference_rebinding`` is an evaluation quirk and does not apply).  A query's history is empty, and its s_h zero,
        when its entity's test-time history is: unlike predict, a forecast has no ground-truth history of the caller's to
        consult.

        ``known``: triples (or quadruples) whose answers are left out of the lists -- every answer known for (e, r), or with
        ``time_aware=True`` (quadruples) only those known at the query's own timestamp.  The excluded answers stay in the
        softmax's normaliser, so a value is the model's probability of its answer; a query with fewer than k admissible
        answers gets id -1 and value 0 in its last slots.

        ``process_group``: sharded as evaluate_stream_batched shards -- roll-over and encoding chunks round-robin,
        contiguous row slices of each top-k call, each rank building its own rows' lists -- and every rank returns the
        one-process result bit for bit (a row's top-k depends on that row alone).  Ranks called with different arguments
        raise ValueError.

        A model on the host takes the same control flow with _encode_one per query, materialised logits and a stable
        sort (topk_excluding_torch)."""
        return self._forecast_stream(self._forecast_queries(queries, k, 'forecast'), global_model, k, subject, known,
                                     time_aware, process_group, 'forecast')

    def forecast_relations(self, queries, global_model, k=10, subject=True, known=None, time_aware=False,
                           process_group=None):
        """The model's k most likely next relations of each entity, over its own test-time state: the relation head's
        p(r | e, history) = softmax(linear_r([ent_e | s_q])), the distribution pred_r_rank2 weighs the roll-over's
        candidates with (model.py:202-208).

        ``queries``: int64 [n, 2] rows (entity, timestamp), timestamps non-decreasing and not before ``latest_time``.
        ``subject=True`` asks which relation e takes part in next as a subject, (e, ?, ., t), from its subject-side
        test-time history; ``False`` as an object, (., ?, e, t), from its object-side history.  Returns (values float32
        [n, k], relation ids int64 [n, k]) on the model's device, p = softmax over all num_rels relations, descending, ties
        to the lower id; an empty history gives a zero s_q (model.py:187-189).  ``known``: triples (or quadruples with
        ``time_aware``) whose relations are left out of each entity's list -- every relation of a known (e, r, .) (or
        (., r, e)), or only those known at the query's own t -- but not out of the softmax; a row with fewer than k
        admissible relations ends in id -1 and value 0.

        forecast's contract otherwise: each timestamp change rolls over through the same _roll_over, leaving the same
        state and RNG stream as forecast; ``process_group`` shards the encoding chunks and top-k rows in the same way and
        every rank returns the one-process result bit for bit.  s_q does not depend on the relation, so each distinct
        entity of a run is encoded once, and the rows are scored by one renet_decoder_topk call against ``linear_r``."""
        return self._forecast_stream(self._forecast_queries(queries, k, 'forecast_relations', relations=True), global_model,
                                     k, subject, known, time_aware, process_group, 'forecast_relations')

    def _forecast_stream(self, qn, global_model, k, subject, known, time_aware, process_group, caller):
        """forecast (qn int64 [n, 3] of (entity, relation, timestamp)) or forecast_relations (qn [n, 2] of (entity,
        timestamp)) over the test-time state, after _forecast_queries' checks; ValueErrors name ``caller``."""
        relation = qn.shape[1] == 2
        q = torch.from_numpy(qn)
        n = len(qn)
        if n and (np.any(np.diff(qn[:, -1]) < 0) or qn[0, -1] < int(self.latest_time)):
            raise ValueError('%s: timestamps must be non-decreasing and not before latest_time = %d'
                             % (caller, int(self.latest_time)))
        if time_aware and known is None:
            raise ValueError('%s: time_aware needs known quadruples (s, r, o, t)' % caller)
        shard = self._eval_shard(process_group, caller)
        if shard is not None:
            import hashlib
            digest = int.from_bytes(hashlib.blake2b(np.ascontiguousarray(qn).tobytes(), digest_size=7).digest(), 'little')
            fp = [n, digest, int(self.latest_time), int(self.num_k), int(k), int(bool(subject)), int(bool(time_aware)),
                  -1 if known is None else len(known)]
            if not shard.same_everywhere(fp):
                raise ValueError('%s: the ranks of process_group were called with different queries, latest_time, '
                                 'num_k, k or flags' % caller)
        self._trim_test_histories()
        index, col = self._forecast_index(known, time_aware, subject, relation, True)
        hist = self.s_hist_test if subject else self.o_hist_test
        dev = self.ent_embeds.device
        values = torch.empty(n, k, device=dev)
        ids = torch.empty(n, k, dtype=torch.long, device=dev)
        with torch.no_grad():
            i0 = 0
            while i0 < n:
                i1 = i0 + 1
                while i1 < n and qn[i1, -1] == qn[i0, -1]:
                    i1 += 1
                t = q[i0, -1]
                if self.latest_time != t:
                    self._roll_over(t, global_model, shard)
                e, r = qn[i0:i1, 0], (None if relation else qn[i0:i1, 1])      # the relation head takes no relation
                has = np.asarray([len(hist[x]) != 0 for x in e], dtype=bool)
                state = self._encode_queries(e, r, has, subject, shard, relation=relation)
                x = self._forecast_rows(e, r, state, subject, relation)
                # a row's top-k depends on that row alone (no split-K, no kernel choice by row count, per-row steps after
                # the GEMM), so a shard scores a contiguous slice of the rows with the lists of its rows only
                m = i1 - i0
                lo, hi = (0, m) if shard is None else shard.slice(m)
                exclude = self._forecast_exclude(index, col, subject, relation, e[lo:hi], None if relation else r[lo:hi],
                                                 np.full(hi - lo, int(t)) if time_aware else None)
                v, c = self._topk_rows(x[lo:hi], k, exclude, self.linear_r if relation else None)
                if shard is not None:
                    v, c = shard.allgather_slices(v, m), shard.allgather_slices(c, m)
                values[i0:i1], ids[i0:i1] = v, c
                i0 = i1
        return values, ids

    def _forecast_index(self, known, time_aware, subject, relation, check_quadruples=False):
        """(index, col) of a forecast's known facts: a FilterIndex / TimeFilterIndex (a RelationFilterIndex for the relation
        head) and its column array for the queried side, on the model's device when it is a GPU (sent once per call; each
        chunk sends its ranges), or (None, None) without ``known``."""
        if known is None:
            return None, None
        if time_aware and check_quadruples:
            known = _quadruples(known)
        if relation:
            index = RelationFilterIndex(known, time_aware)
            col = index.col(subject)
        else:
            index = TimeFilterIndex(known) if time_aware else FilterIndex(known)
            col = index.col('objects' if subject else 'subjects')
        if self.ent_embeds.is_cuda:
            col = torch.from_numpy(col).to(self.ent_embeds.device)
        return index, col

    def _forecast_rows(self, e, r, state, subject, relation):
        """The decoder rows of forecast queries with entities e and relations r (host arrays) and their encoder states:
        [ent_e | s_h | rel_r] for the entity head (inverse relation embeddings for subject=False), [ent_e | s_q] for the
        relation head."""
        dev = self.ent_embeds.device
        ent = self.ent_embeds[torch.from_numpy(e).to(dev)]
        if relation:
            return torch.cat((ent, state), dim=1)
        rel_embeds, _ = self._direction(subject)
        return torch.cat((ent, state, rel_embeds[torch.from_numpy(r).to(dev)]), dim=1)

    def _forecast_exclude(self, index, col, subject, relation, e, r, t):
        """(col, begin, end) of forecast rows with entities e, relations r and, time-aware, timestamps t (else None), or
        None without an index."""
        if index is None:
            return None
        tt = () if t is None else (t,)
        if relation:
            return (col,) + index.ranges(subject, e, *tt)
        return (col,) + index.ranges('objects' if subject else 'subjects', e, r, *tt)

    def _forecast_queries(self, queries, k, caller, relations=False):
        """The forecast calls' checks on ``queries`` (integer rows (entity, relation, timestamp), ids in range; with
        ``relations``, rows (entity, timestamp)) and ``k`` (at most the number of answers: entities, or relations with
        ``relations``); ValueErrors name ``caller``.  Returns the queries as a host int64 array [n, 3] ([n, 2])."""
        from .decoder import TOPK_MAX_K
        q = torch.as_tensor(queries)
        cols, what = (2, '(entity, timestamp)') if relations else (3, '(entity, relation, timestamp)')
        if q.dim() != 2 or q.shape[1] != cols or q.dtype.is_floating_point:
            raise ValueError('%s: queries must be integer rows %s, got %s %s' % (caller, what, tuple(q.shape), q.dtype))
        qn = q.cpu().long().numpy()
        n = len(qn)
        top = min(self.num_rels if relations else self.in_dim, TOPK_MAX_K)
        if not 1 <= k <= top:
            raise ValueError('%s: k = %d outside [1, %d]' % (caller, k, top))
        if n and (qn[:, 0].min() < 0 or qn[:, 0].max() >= self.in_dim):
            raise ValueError('%s: entity ids outside [0, %d)' % (caller, self.in_dim))
        if not relations and n and (qn[:, 1].min() < 0 or qn[:, 1].max() >= self.num_rels):
            raise ValueError('%s: relation ids outside [0, %d)' % (caller, self.num_rels))
        return qn

    def forecast_observed(self, queries, history, graph_dict, global_emb, k=10, subject=True, known=None,
                          time_aware=False):
        """The model's k most likely answers of each query over observed history: forecast's result for queries whose
        histories the caller knows, as evaluate_observed encodes a test triple from its own history.

        ``queries``: int64 [n, 3] rows (entity, relation, timestamp), in any order.  ``history`` = (lists, timestamp lists),
        one entry per query: the entity's subject-side history for ``subject=True``, its object-side one otherwise, in the
        format evaluate_observed takes (e.g. synthetic.observed_history of the known facts).  Every timestamp of a query's
        history must be before the query's own timestamp.  ``graph_dict`` / ``global_emb``: the true graphs and global
        embeddings of the timestamps those histories reference, as evaluate_observed takes them.

        Returns forecast's result: (values float32 [n, k], entity ids int64 [n, k]) on the model's device, p = softmax over
        all entities, descending, ties to the lower id.  ``subject=True`` scores the objects of (e, r, ?, t) from
        [ent_e | s_h | rel_r], ``False`` the subjects of (?, r, e, t) with the inverse relation embeddings; an empty history
        gives a zero s_h.  ``known``: triples whose answers are left out of the lists but not out of the normaliser, or
        with ``time_aware=True`` quadruples, of which only the answers known at the query's own t are left out.  A row
        with fewer than k admissible answers ends in id -1 and value 0.

        Nothing rolls over, nothing is sampled and the global model is not called: the test-time state, graph_dict,
        global_emb, latest_time and torch's RNG stay as they were.  The model scores in eval mode and its mode is restored.
        The distinct (entity, relation, history) queries are encoded once by _encode_queries (each (entity, timestamp)
        component built once), and the rows are scored OBSERVED_RANK_ROWS at a time by renet_decoder_topk with one
        exclusion list per row from a FilterIndex / TimeFilterIndex built once per call; a row's top-k depends on that row
        alone, so the chunk size changes no bit.  Every ValueError -- evaluate_observed's checks on the histories, forecast's
        on ``queries`` and ``k``, a history timestamp not before its query's -- comes before any work.  A model on the host
        takes the same flow through _encode_one, ``linear`` and topk_excluding_torch."""
        return self._forecast_from_history(self._forecast_queries(queries, k, 'forecast_observed'), history, graph_dict,
                                           global_emb, k, subject, known, time_aware, 'forecast_observed')

    def forecast_relations_observed(self, queries, history, graph_dict, global_emb, k=10, subject=True, known=None,
                                    time_aware=False):
        """The model's k most likely next relations of each entity over observed history: forecast_relations' result for
        queries whose histories the caller knows, with forecast_observed's arguments and guarantees.

        ``queries``: int64 [n, 2] rows (entity, timestamp), in any order.  ``history``: one window per query, the entity's
        subject-side history for ``subject=True`` and its object-side one otherwise (e.g. synthetic.observed_history of the
        known facts), every timestamp before the query's own.  Returns (values float32 [n, k], relation ids int64 [n, k]),
        p = softmax(linear_r([ent_e | s_q])) over all num_rels relations, descending, ties to the lower id; an empty history
        gives a zero s_q.  ``known`` (triples, or quadruples with ``time_aware``) leaves the entity's known relations on
        that side out of the list but not out of the softmax; a row with fewer than k admissible relations ends in id -1
        and value 0.

        Nothing rolls over, nothing is sampled, the global model is not called, and the state, RNG and module mode are
        left as they were.  Each distinct (entity, history) is encoded once by _encode_queries, and the rows are scored
        OBSERVED_RANK_ROWS at a time by renet_decoder_topk against ``linear_r``.  Every ValueError comes before any work."""
        return self._forecast_from_history(self._forecast_queries(queries, k, 'forecast_relations_observed', relations=True),
                                           history, graph_dict, global_emb, k, subject, known, time_aware,
                                           'forecast_relations_observed')

    def _forecast_from_history(self, qn, history, graph_dict, global_emb, k, subject, known, time_aware, caller):
        """forecast_observed (qn int64 [n, 3] of (entity, relation, timestamp)) or forecast_relations_observed (qn [n, 2] of
        (entity, timestamp)) after _forecast_queries' checks; ValueErrors name ``caller``."""
        relation = qn.shape[1] == 2
        n = len(qn)
        if len(history) != 2 or len(history[0]) != n or len(history[1]) != n:
            raise ValueError('%s: history must be (lists, timestamp lists) of %d queries' % (caller, n))
        if known is not None:
            kt = torch.as_tensor(known)
            if kt.dim() != 2 or kt.shape[1] < (4 if time_aware else 3):
                raise ValueError('%s: known must be %s' % (caller, 'quadruples (s, r, o, t) with time_aware'
                                                           if time_aware else 'triples (s, r, o)'))
        elif time_aware:
            raise ValueError('%s: time_aware needs known quadruples (s, r, o, t)' % caller)
        obs, has = self._observed_histories(qn[:, 0], history, 'history', graph_dict, global_emb, before=qn[:, -1],
                                            caller=caller)
        index, col = self._forecast_index(known, time_aware, subject, relation)
        dev = self.ent_embeds.device
        values = torch.empty(n, k, device=dev)
        ids = torch.empty(n, k, dtype=torch.long, device=dev)
        modes = [(mod, mod.training) for mod in self.modules()]
        self.eval()
        try:
            with torch.no_grad():
                rels = None if relation else qn[:, 1]                           # the relation head takes no relation
                state = self._encode_queries(qn[:, 0], rels, has, subject, history=obs, graphs=(graph_dict, global_emb),
                                             relation=relation)
                for i0 in range(0, n, OBSERVED_RANK_ROWS):
                    i1 = min(i0 + OBSERVED_RANK_ROWS, n)
                    e, r = qn[i0:i1, 0], (None if relation else rels[i0:i1])
                    x = self._forecast_rows(e, r, state[i0:i1], subject, relation)
                    exclude = self._forecast_exclude(index, col, subject, relation, e, r,
                                                     qn[i0:i1, -1] if time_aware else None)
                    values[i0:i1], ids[i0:i1] = self._topk_rows(x, k, exclude, self.linear_r if relation else None)
        finally:
            for mod, mode in modes:
                mod.training = mode
        return values, ids

    def _topk_rows(self, x, k, exclude, linear=None):
        """(values [M, k], ids int64 [M, k]) of the rows of x against ``linear`` (the entity head's unless another is given)
        with the exclusion lists ``exclude`` = (col, begin, end) or None: one renet_decoder_topk call on the GPU; on the
        host, row by row through ``linear`` as predict computes them, then topk_excluding_torch."""
        from .decoder import decoder_topk
        linear = self.linear if linear is None else linear
        dev = x.device
        if len(x) == 0:                  # a shard without rows: the empty results keep the dtypes the all-gather needs
            return torch.zeros(0, k, device=dev), torch.zeros(0, k, dtype=torch.long, device=dev)
        if x.is_cuda:
            ex = None
            if exclude is not None:
                ex = (exclude[0],) + tuple(torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(dev)
                                           for a in exclude[1:])
            return decoder_topk(x, linear.weight, linear.bias, k, ex)
        z = torch.stack([linear(row) for row in x])
        return topk_excluding_torch(z, k, exclude)

