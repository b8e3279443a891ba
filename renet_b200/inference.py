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


#: distinct (entity, timestamp) components evaluate_stream_batched batches per chunk are bounded by their summed node and
#: candidate-edge counts: the plan's mark_off / cand_off are int32, and 2^28 keeps them far from overflow
EVAL_PLAN_BUDGET = 1 << 28


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

    def _encode_one(self, entity, r, history, history_t, subject):
        """Final hidden state of `encoder` for ONE (entity, relation) history (aggregator.predict + encoder,
        model.py:333-351)."""
        rel_embeds, reverse = self._direction(subject)
        dev = self.ent_embeds.device
        e = torch.as_tensor(entity, device=dev).view(1)
        rr = torch.as_tensor(r, device=dev).view(1)
        s_h, _, _ = self.aggregator.encode(([history], [history_t]), e, rr, self.ent_embeds, rel_embeds, self.graph_dict,
                                           self.global_emb, reverse, self.encoder, self.encoder_r)
        return s_h.view(-1)

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
        from .hoststore import GraphStore, HistoryStore
        hist = self.s_hist_test if subject else self.o_hist_test
        hist_t = self.s_hist_test_t if subject else self.o_hist_test_t
        times = sorted({int(t) for e in entities for t in hist_t[e]})
        gs = GraphStore({t: self.graph_dict[t] for t in times})
        store = HistoryStore([hist[e] for e in entities], [hist_t[e] for e in entities], entities, gs, dedupe=False)
        samples = np.asarray(samples, dtype=np.int64)
        return store.select(samples, groups=samples), gs

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
        """[c0, c1) of pred_r_topk's chunks of n entities: ROLLOVER_SEQ_BUDGET // R entities each."""
        per = max(1, ROLLOVER_SEQ_BUDGET // self.num_rels)
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
        from .decoder import ranks_from_counts
        R, h = self.num_rels, self.h_dim
        dev = self.ent_embeds.device
        n = len(quads)
        s, r, o = quads[:, 0].copy(), quads[:, 1].copy(), quads[:, 2].copy()
        si, oi = s.copy(), o.copy()
        if rebind is not None:
            si[0], oi[0] = rebind
        has_s = ~s_empty & np.asarray([len(self.s_hist_test[e]) != 0 for e in si], dtype=bool)
        has_o = ~o_empty & np.asarray([len(self.o_hist_test[e]) != 0 for e in oi], dtype=bool)
        s_h = self._encode_queries(si, r, has_s, True, shard)
        o_h = self._encode_queries(oi, r, has_o, False, shard)
        to_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to(dev)    # noqa: E731
        si_d, oi_d, r_d = to_dev(si), to_dev(oi), to_dev(r)
        x = torch.cat((torch.cat((self.ent_embeds[si_d], s_h, self.rel_embeds[:R][r_d]), dim=1),
                       torch.cat((self.ent_embeds[oi_d], o_h, self.rel_embeds[R:][r_d]), dim=1)), dim=0)
        rank_lab = np.concatenate((o, s))                        # ob rows rank the triple's object, sub rows its subject
        loss_row = np.concatenate((np.arange(n), n + np.arange(n)))
        if rebind is not None and (si[0] != s[0] or oi[0] != o[0]):
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
                excludes.append(_exclusion_lists(tfidx, direction, fix, rr, np.full(hi - lo, quads[0, 3])))
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

    def _rank_rows(self, x, label, excludes):
        """(loss_rows [M], counts [M, 2 + 2L]) of the rows of x against ``linear``: the raw (greater, equal) pair, then the
        filtered pair against each of the L = 0-2 exclusion lists ``excludes``.  One renet_decoder_rank_multi call on the
        GPU; on the host, row by row through ``linear`` as predict computes them, counted with torch once per list."""
        from .decoder import decoder_rank_counts_multi
        dev = x.device
        lab = torch.from_numpy(np.ascontiguousarray(label, dtype=np.int64)).to(dev)
        if len(lab) == 0:
            # a shard without rows (fewer rows than ranks): nothing to launch, and the empty results keep the dtypes of
            # the other ranks' shares, which the all-gather after this call needs
            return (torch.zeros(0, device=dev),
                    torch.zeros(0, 2 + 2 * len(excludes), dtype=torch.int32 if x.is_cuda else torch.long, device=dev))
        if x.is_cuda:
            ex = [tuple(torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(dev) for a in e) for e in excludes]
            return decoder_rank_counts_multi(x, self.linear.weight, self.linear.bias, lab, ex)
        z = torch.stack([self.linear(row) for row in x])
        loss_rows = torch.stack([self.criterion(z[m].view(1, -1), lab[m].view(1)) for m in range(len(lab))])
        cs = [rank_counts_torch(z, lab, e) for e in excludes]
        return loss_rows, torch.cat([rank_counts_torch(z, lab)[:, :2]] + [ci[:, 2:] for ci in cs], dim=1)

    def _encode_queries(self, ents, rels, has, subject, shard=None):
        """s_h [n, h] of the queries (ents[i], rels[i]) against the current test-time histories; rows where ``has`` is
        False stay zero (predict's empty-history rule).  Equal queries are encoded once.  On the GPU the distinct queries go
        through the device batcher in chunks, one isolation group per entity, so that each equals _encode_one's encoding
        of it alone; on the host, through _encode_one, one query per chunk.  With a ``shard`` chunk j runs on rank
        j mod world and every rank all-gathers the encodings."""
        h, R = self.h_dim, self.num_rels
        dev = self.ent_embeds.device
        out = torch.zeros(len(ents), h, device=dev)
        sel = np.flatnonzero(has)
        if len(sel) == 0:
            return out
        keys, inverse = np.unique(np.asarray(ents)[sel].astype(np.int64) * R + np.asarray(rels)[sel], return_inverse=True)
        q_e, q_r = keys // R, keys % R
        hist = self.s_hist_test if subject else self.o_hist_test
        hist_t = self.s_hist_test_t if subject else self.o_hist_test_t
        if not self.ent_embeds.is_cuda:
            chunks = [(j, j + 1) for j in range(len(keys))]
        else:
            rel_embeds, reverse = self._direction(subject)
            sizes = {}
            for t in {int(t) for e in np.unique(q_e) for t in hist_t[e]}:
                g = self.graph_dict[t]
                sizes[t] = g.number_of_nodes() + g.number_of_edges()
            chunks, j0 = [], 0
            while j0 < len(keys):
                # a chunk: whole entities (keys are sorted by entity), within both budgets
                cost, j1 = 0, j0
                while j1 < len(keys) and j1 - j0 < ROLLOVER_SEQ_BUDGET:
                    e = q_e[j1]
                    if j1 == j0 or e != q_e[j1 - 1]:
                        c = sum(sizes[int(t)] for t in hist_t[e])
                        if j1 > j0 and cost + c > EVAL_PLAN_BUDGET:
                            break
                        cost += c
                    j1 += 1
                chunks.append((j0, j1))
                j0 = j1
        parts = []
        for j0, j1 in (chunks[c] for c in (range(len(chunks)) if shard is None else shard.units(len(chunks)))):
            if not self.ent_embeds.is_cuda:
                e, rr = int(q_e[j0]), int(q_r[j0])
                parts.append(self._encode_one(e, rr, hist[e], hist_t[e], subject).view(1, h).to(out.dtype))
                continue
            ue, pos = np.unique(q_e[j0:j1], return_inverse=True)
            view, gs = self._grouped_view(ue, pos, subject)
            s_dev = torch.from_numpy(q_e[j0:j1]).to(dev)
            r_dev = torch.from_numpy(q_r[j0:j1]).to(dev)
            sh, _, hb = self.aggregator.encode(view, s_dev, r_dev, self.ent_embeds, rel_embeds, gs, self.global_emb,
                                               reverse, self.encoder, self.encoder_r)
            # the encoder returns the sequences length-sorted: row k is sample sample_order[k] of the view
            idx = hb.sample_order(dev)
            part = torch.empty_like(sh)
            part[idx] = sh
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
        from .decoder import TOPK_MAX_K
        q = torch.as_tensor(queries)
        if q.dim() != 2 or q.shape[1] != 3 or q.dtype.is_floating_point:
            raise ValueError('forecast: queries must be integer rows (entity, relation, timestamp), got %s %s'
                             % (tuple(q.shape), q.dtype))
        q = q.cpu().long()
        qn = q.numpy()
        n = len(qn)
        if not 1 <= k <= min(self.in_dim, TOPK_MAX_K):
            raise ValueError('forecast: k = %d outside [1, %d]' % (k, min(self.in_dim, TOPK_MAX_K)))
        if n and (qn[:, 0].min() < 0 or qn[:, 0].max() >= self.in_dim):
            raise ValueError('forecast: entity ids outside [0, %d)' % self.in_dim)
        if n and (qn[:, 1].min() < 0 or qn[:, 1].max() >= self.num_rels):
            raise ValueError('forecast: relation ids outside [0, %d)' % self.num_rels)
        if n and (np.any(np.diff(qn[:, 2]) < 0) or qn[0, 2] < int(self.latest_time)):
            raise ValueError('forecast: timestamps must be non-decreasing and not before latest_time = %d'
                             % int(self.latest_time))
        if time_aware and known is None:
            raise ValueError('forecast: time_aware needs known quadruples (s, r, o, t)')
        shard = self._eval_shard(process_group, 'forecast')
        if shard is not None:
            import hashlib
            digest = int.from_bytes(hashlib.blake2b(np.ascontiguousarray(qn).tobytes(), digest_size=7).digest(), 'little')
            fp = [n, digest, int(self.latest_time), int(self.num_k), int(k), int(bool(subject)), int(bool(time_aware)),
                  -1 if known is None else len(known)]
            if not shard.same_everywhere(fp):
                raise ValueError('forecast: the ranks of process_group were called with different queries, latest_time, '
                                 'num_k, k or flags')
        self._trim_test_histories()
        index = None
        if known is not None:
            index = TimeFilterIndex(_quadruples(known)) if time_aware else FilterIndex(known)
        dev = self.ent_embeds.device
        direction = 'objects' if subject else 'subjects'
        col = None
        if index is not None:
            col = index.col(direction)
            if self.ent_embeds.is_cuda:
                col = torch.from_numpy(col).to(dev)                  # once per call; each run sends its ranges
        rel_embeds, _ = self._direction(subject)
        hist = self.s_hist_test if subject else self.o_hist_test
        values = torch.empty(n, k, device=dev)
        ids = torch.empty(n, k, dtype=torch.long, device=dev)
        with torch.no_grad():
            i0 = 0
            while i0 < n:
                i1 = i0 + 1
                while i1 < n and qn[i1, 2] == qn[i0, 2]:
                    i1 += 1
                t = q[i0, 2]
                if self.latest_time != t:
                    self._roll_over(t, global_model, shard)
                e, r = qn[i0:i1, 0], qn[i0:i1, 1]
                has = np.asarray([len(hist[x]) != 0 for x in e], dtype=bool)
                s_h = self._encode_queries(e, r, has, subject, shard)
                x = torch.cat((self.ent_embeds[torch.from_numpy(e).to(dev)], s_h, rel_embeds[torch.from_numpy(r).to(dev)]),
                              dim=1)
                # a row's top-k depends on that row alone (no split-K, no kernel choice by row count, per-row steps after
                # the GEMM), so a shard scores a contiguous slice of the rows with the lists of its rows only
                m = i1 - i0
                lo, hi = (0, m) if shard is None else shard.slice(m)
                exclude = None
                if index is not None:
                    key = (e[lo:hi], r[lo:hi]) + ((np.full(hi - lo, int(t)),) if time_aware else ())
                    exclude = (col,) + index.ranges(direction, *key)
                v, c = self._topk_rows(x[lo:hi], k, exclude)
                if shard is not None:
                    v, c = shard.allgather_slices(v, m), shard.allgather_slices(c, m)
                values[i0:i1], ids[i0:i1] = v, c
                i0 = i1
        return values, ids

    def _topk_rows(self, x, k, exclude):
        """(values [M, k], ids int64 [M, k]) of the rows of x against ``linear`` with the exclusion lists ``exclude`` =
        (col, begin, end) or None: one renet_decoder_topk call on the GPU; on the host, row by row through ``linear`` as
        predict computes them, then topk_excluding_torch."""
        from .decoder import decoder_topk
        dev = x.device
        if len(x) == 0:                  # a shard without rows: the empty results keep the dtypes the all-gather needs
            return torch.zeros(0, k, device=dev), torch.zeros(0, k, dtype=torch.long, device=dev)
        if x.is_cuda:
            ex = None
            if exclude is not None:
                ex = (exclude[0],) + tuple(torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(dev)
                                           for a in exclude[1:])
            return decoder_topk(x, self.linear.weight, self.linear.bias, k, ex)
        z = torch.stack([self.linear(row) for row in x])
        return topk_excluding_torch(z, k, exclude)

