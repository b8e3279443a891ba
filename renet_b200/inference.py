"""Test-time path of RE-Net on the H100 kernels (reference model.py:107-446; SURVEY.md section 8(f) row 2).

``RENetInference`` is mixed into ``renet_b200.model.RENet`` and provides the reference's evaluation API --
``init_history``, ``pred_r_rank2``, ``predict``, ``evaluate``, ``evaluate_filter``, ``update_cache`` -- with the same
arguments, return values and state attributes (``s_hist_test``, ``s_his_cache``, ``latest_time``, ``graph_dict``,
``global_emb`` ...), so the reference's ``test.py`` / validation loop (train.py:151-185) drive it unchanged.

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

    def pred_r_topk(self, entities, weights, k, subject=True, capacity=None):
        """pred_r_rank2 followed by torch.topk for many entities at once (model.py:168-213, 236-240).  For entity
        entities[i]: the k largest entries of weights[i] * pred_r_rank2([entities[i]] * R, arange(R), subject).view(-1)
        and their codes r * in_dim + o, as (values float32 [n, k], codes int64 [n, k]) on the model's device.

        The test-time histories of a chunk of entities are encoded in one batched call (one store entry per entity, each
        repeated once per relation, through the C++ / device batcher, over a graph store built for the chunk in which
        every entity has its own copies of its history's graphs); entities without history get zero s_h / s_q as in
        pred_r_rank2.  The joint distribution is never materialised: renet_decoder_group_topk scores
        [ent_e | s_h(e, r) | rel_r] against ``linear`` with the row weights weights[i] * softmax_r(linear_r([ent_e | s_q_e]))
        and selects each entity's k best in one pass.  A group's k entries come in the order torch.topk(sorted=False) gives
        on a CUDA tensor of R * in_dim values (ORDER_INDEX: the values above the k-th one in index order, then those equal
        to it; measured on an H100 with PyTorch 2.11 from R * in_dim = 9 600 to 5.9 M), since the roll-over's final
        selection and the order of its cache updates depend on that layout."""
        from .decoder import ORDER_INDEX, decoder_group_topk
        from .hoststore import GraphStore, HistoryStore
        R, h, N = self.num_rels, self.h_dim, self.in_dim
        dev = self.ent_embeds.device
        ents = torch.as_tensor(entities).reshape(-1).long().cpu().numpy()
        wts = torch.as_tensor(weights).reshape(-1).to(device=dev, dtype=torch.float32)
        n = len(ents)
        if wts.numel() != n:
            raise ValueError('pred_r_topk: %d entities but %d weights' % (n, wts.numel()))
        values = torch.empty(n, k, device=dev)
        codes = torch.empty(n, k, dtype=torch.long, device=dev)
        rel_embeds, reverse = self._direction(subject)
        hist = self.s_hist_test if subject else self.o_hist_test
        hist_t = self.s_hist_test_t if subject else self.o_hist_test_t
        per = max(1, ROLLOVER_SEQ_BUDGET // R)
        rel_rows = torch.arange(R, device=dev)
        for c0 in range(0, n, per):
            ce = ents[c0:c0 + per]
            nc = len(ce)
            s_h = torch.zeros(nc, R, h, device=dev)
            s_q = torch.zeros(nc, h, device=dev)
            has = np.flatnonzero([len(hist[e]) != 0 for e in ce])
            if len(has):
                he = ce[has]
                # The batched history graph has one component per timestamp, induced by the nodes of every sample in
                # the batch (utils.py:158-181), so an entity's encoding depends on what it is batched with.  Each entity
                # gets its own copies of its history's graphs, under keys of its own, to encode exactly what
                # pred_r_rank2 encodes alone.
                span = max(len(hist_t[e]) for e in he)
                keys = [[j * span + i for i in range(len(hist_t[e]))] for j, e in enumerate(he)]
                graphs, glob = {}, {}
                for e, ks in zip(he, keys):
                    for v, t in zip(ks, hist_t[e]):
                        graphs[v], glob[v] = self.graph_dict[int(t)], self.global_emb[int(t)]
                gs = GraphStore(graphs)
                store = HistoryStore([hist[e] for e in he], keys, he, gs, dedupe=False)
                view = store.select(np.repeat(np.arange(len(he)), R))
                s_dev = torch.from_numpy(np.repeat(he, R)).to(dev)
                r_dev = rel_rows.repeat(len(he))
                sh, sq, hb = self.aggregator.encode(view, s_dev, r_dev, self.ent_embeds, rel_embeds, gs, glob, reverse,
                                                    self.encoder, self.encoder_r)
                # the encoder returns the sequences length-sorted: row j is sample sample_order[j] of the view
                idx = hb.sample_order(dev)
                sh_v, sq_v = torch.empty_like(sh), torch.empty_like(sq)
                sh_v[idx], sq_v[idx] = sh, sq
                has_dev = torch.from_numpy(has).to(dev)
                s_h[has_dev] = sh_v.view(len(he), R, h)
                s_q[has_dev] = sq_v.view(len(he), R, h)[:, 0]                 # s_q does not depend on r (model.py:96)
            ent = self.ent_embeds[torch.from_numpy(ce).to(dev)]
            p_r = torch.softmax(self.linear_r(torch.cat((ent, s_q), dim=1)), dim=1)                    # [nc, R]
            row_w = (wts[c0:c0 + nc].view(-1, 1) * p_r).reshape(-1)
            x = torch.cat((ent.repeat_interleave(R, dim=0), s_h.view(nc * R, h), rel_embeds.repeat(nc, 1)), dim=1)
            v, i = decoder_group_topk(x, self.linear.weight, self.linear.bias, row_w, R, k, ORDER_INDEX, capacity)
            values[c0:c0 + nc] = v
            codes[c0:c0 + nc] = i
        return values, codes

    def _pick_candidates(self, picks, prob, subject):
        """The num_k most probable (relation, entity) continuations of every pick (model.py:236-240): host tensors
        (joint probabilities [n_picks, num_k], codes r * in_dim + o [n_picks, num_k]) in picks order.  On the GPU every
        distinct entity is scored once, all of them in one batched pass (pred_r_topk: its scores depend on the entity
        only), and its list is repeated for each pick of it.  A model on the host has no kernels to run (the host-logic
        checks substitute a host encoder): its picks are scored one by one through pred_r_rank2, as the reference does."""
        K, R = self.num_k, self.num_rels
        if self.ent_embeds.is_cuda:
            uniq, inverse = torch.unique(picks, return_inverse=True)
            top_p, top_i = self.pred_r_topk(uniq, prob[uniq], K, subject=subject)
            inverse = inverse.cpu()
            return top_p.cpu()[inverse], top_i.cpu()[inverse]
        lists, inds = [], []
        for e, p_e in zip(picks, prob[picks]):
            ee = torch.full((R,), int(e), dtype=torch.long)
            joint = float(p_e) * self.pred_r_rank2(ee, torch.arange(R), subject=subject)
            top_p, top_i = torch.topk(joint.view(-1), K, sorted=False)
            lists.append(top_p.view(-1).cpu())
            inds.append(top_i.view(-1).cpu())
        return torch.stack(lists), torch.stack(inds)

    def _roll_over(self, t, global_model):
        """model.py:222-330: the stream moved to a new timestamp.  Sample num_k subjects (objects) from the global
        model's distribution, score every (relation, entity) continuation for them, keep the num_k most probable
        triples, turn them into the predicted graph of `latest_time`, and roll the per-entity histories."""
        K, R = self.num_k, self.num_rels
        last = {}
        for subject in (True, False):
            cache = self.s_his_cache if subject else self.o_his_cache
            cache_t = self.s_his_cache_t if subject else self.o_his_cache_t
            if subject:
                _, _, prob = global_model.predict(self.latest_time, self.graph_dict, subject=True)
            else:
                _, logits, _ = global_model.predict(t, self.graph_dict, subject=False)
                prob = torch.softmax(logits.view(-1), dim=0)                               # model.py:262
            picks = torch.distributions.categorical.Categorical(prob).sample(torch.Size([K]))
            # NOTE: the reference de-duplicates with a set of 0-dim tensors (model.py:228-234), which never matches
            # (tensors hash by identity), so repeated samples are scored again and kept as separate entries.
            lists, inds = self._pick_candidates(picks, prob, subject)                     # [K picks, K] in picks order
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
        s, r, o = int(triplet[0]), int(triplet[1]), int(triplet[2])
        loss, sub_pred, ob_pred = self.predict(triplet, s_hist, o_hist, global_model)
        sub_pred, ob_pred = torch.sigmoid(sub_pred), torch.sigmoid(ob_pred)
        allt = torch.as_tensor(all_triplets).to(ob_pred.device)
        ranks = []
        for pred, label, col_fix, col_out, fix in ((sub_pred, s, 2, 0, o), (ob_pred, o, 0, 2, s)):
            ground = pred[label].clone()
            known = allt[(allt[:, col_fix] == fix) & (allt[:, 1] == r)][:, col_out].long()
            pred = pred.clone()
            pred[known] = 0
            pred[label] = ground
            ranks.append(rank_with_ties(pred, label))
        return np.array(ranks), loss

    def evaluate_stream(self, test_data, s_history, o_history, global_model, total_data=None, raw=False):
        """The reference's test loop (test.py:98-150) as a method: trims the per-entity histories to ``seq_len``
        (test.py:100-106), ranks every test triple in stream order (``evaluate`` when ``raw`` else ``evaluate_filter``
        against ``total_data``), and returns MRR / MR / Hits@{1,3,10} over subject and object ranks together, the summed
        loss and the ranks.  ``s_history`` / ``o_history`` = (lists, timestamp lists) of the test split."""
        for hist, hist_t in ((self.s_hist_test, self.s_hist_test_t), (self.o_hist_test, self.o_hist_test_t)):
            for ee in range(self.in_dim):
                while len(hist[ee]) > self.seq_len:
                    hist[ee].pop(0)
                    hist_t[ee].pop(0)
        test_data = torch.as_tensor(test_data)
        if not raw:
            if total_data is None:
                raise ValueError('filtered evaluation needs total_data (all known triples)')
            total_data = torch.as_tensor(total_data).to(self.ent_embeds.device)
        ranks, total_loss = [], 0.0
        with torch.no_grad():
            for i in range(len(test_data)):
                trip = test_data[i].to(self.ent_embeds.device)
                sh, oh = (s_history[0][i], s_history[1][i]), (o_history[0][i], o_history[1][i])
                if raw:
                    r, loss = self.evaluate(trip, sh, oh, global_model)
                else:
                    r, loss = self.evaluate_filter(trip, sh, oh, global_model, total_data)
                ranks.append(r)
                total_loss += float(loss)
        ranks = np.concatenate(ranks) if ranks else np.zeros(0)
        out = {'mrr': float(np.mean(1.0 / ranks)) if len(ranks) else float('nan'),
               'mr': float(np.mean(ranks)) if len(ranks) else float('nan'), 'loss': total_loss, 'ranks': ranks}
        for k in (1, 3, 10):
            out['hits@%d' % k] = float(np.mean(ranks <= k)) if len(ranks) else float('nan')
        return out

