"""RENet with the reference's class surface (reference model.py:10-104) on the sm_90a kernels.

Constructor signature, attribute and parameter names (``ent_embeds``, ``rel_embeds``, ``encoder``,
``encoder_r``, ``aggregator``, ``linear``, ``linear_r``, ``global_emb``, ``graph_dict`` ...) are the
reference's, so a reference checkpoint's ``state_dict`` loads as is.  ``forward(triplets, s_hist,
o_hist, graph_dict, subject=True) -> loss`` follows model.py:64-104: direction select, sort by
history length, RGCN aggregate, GRU final hidden, zero rows for empty histories, the two linear
decoders + cross-entropy (fused on the wgmma engine, decoder.py: SURVEY.md section 8(f) row 3).

The test-time autoregressive routines (model.py:107-446: ``init_history``, ``pred_r_rank2``,
``predict``, ``evaluate``, ``evaluate_filter``, ``update_cache``) come from ``inference.RENetInference``
(SURVEY.md section 8(f) row 2) and run on the same kernels.
"""
from collections import defaultdict

import torch
import torch.nn as nn

from .aggregator import RGCNAggregator
from .inference import RENetInference


class RENet(RENetInference, nn.Module):
    def __init__(self, in_dim, h_dim, num_rels, dropout=0, model=0, seq_len=10, num_k=10, num_bases=100):
        super(RENet, self).__init__()
        self.in_dim = in_dim
        self.h_dim = h_dim
        self.num_rels = num_rels
        self.model = model
        self.seq_len = seq_len
        self.num_k = num_k
        self.rel_embeds = nn.Parameter(torch.Tensor(2 * num_rels, h_dim))
        nn.init.xavier_uniform_(self.rel_embeds, gain=nn.init.calculate_gain('relu'))
        self.ent_embeds = nn.Parameter(torch.Tensor(in_dim, h_dim))
        nn.init.xavier_uniform_(self.ent_embeds, gain=nn.init.calculate_gain('relu'))

        self.dropout = nn.Dropout(dropout)
        self.encoder = nn.GRU(4 * h_dim, h_dim, batch_first=True)       # parameters only; math is fused
        self.encoder_r = nn.GRU(3 * h_dim, h_dim, batch_first=True)

        self.preds_list_s = defaultdict(lambda: torch.zeros(self.num_k))
        self.preds_ind_s = defaultdict(lambda: torch.zeros(self.num_k))
        self.preds_list_o = defaultdict(lambda: torch.zeros(self.num_k))
        self.preds_ind_o = defaultdict(lambda: torch.zeros(self.num_k))

        # the reference hard-codes num_bases = 100 (model.py:36); exposed only for small test shapes
        self.aggregator = RGCNAggregator(h_dim, dropout, in_dim, num_rels, num_bases, model, seq_len)

        self.linear = nn.Linear(3 * h_dim, in_dim)
        self.linear_r = nn.Linear(2 * h_dim, num_rels)
        self.global_emb = None

        self.s_hist_test = None
        self.o_hist_test = None
        self.s_hist_test_t = None
        self.o_hist_test_t = None
        self.s_his_cache = None
        self.o_his_cache = None
        self.s_his_cache_t = None
        self.o_his_cache_t = None
        self.graph_dict = None
        self.data = None
        self.latest_time = 0
        self.criterion = nn.CrossEntropyLoss()

    def encode(self, triplets, s_hist, o_hist, graph_dict, subject=True):
        """model.py:65-88,94-96: returns (s, r, o) re-ordered by history length, s_h, s_q (zero rows for
        empty histories) and the direction's relation table."""
        if subject:
            rel_embeds = self.rel_embeds[:self.num_rels]
            s, r, o = triplets[:, 0], triplets[:, 1], triplets[:, 2]
            hist, reverse = s_hist, False
        else:
            rel_embeds = self.rel_embeds[self.num_rels:]
            o, r, s = triplets[:, 0], triplets[:, 1], triplets[:, 2]
            hist, reverse = o_hist, True
        s_h, s_q, hb = self.aggregator.encode(hist, s, r, self.ent_embeds, rel_embeds, graph_dict,
                                              self.global_emb, reverse, self.encoder, self.encoder_r, triplets=triplets)
        idx = hb.sample_order(triplets.device)
        if s_h.shape[0] < len(s):                                         # (the no-autograd path pads by itself)
            pad = torch.zeros(len(s) - s_h.shape[0], self.h_dim, device=s_h.device)
            s_h = torch.cat((s_h, pad), dim=0)                            # model.py:88
            s_q = torch.cat((s_q, pad), dim=0)                            # model.py:96
        return s[idx], r[idx], o[idx], s_h, s_q, rel_embeds

    def decode_loss(self, s, r, o, s_h, s_q, rel_embeds):
        """model.py:89-91, 97-103."""
        from .decoder import decoder_cross_entropy
        x = self.dropout(torch.cat((self.ent_embeds[s], s_h, rel_embeds[r]), dim=1))
        loss_sub = decoder_cross_entropy(x, self.linear.weight, self.linear.bias, o)           # fused logits + CE
        x_r = self.dropout(torch.cat((self.ent_embeds[s], s_q), dim=1))
        loss_sub_r = decoder_cross_entropy(x_r, self.linear_r.weight, self.linear_r.bias, r)
        return loss_sub + 0.1 * loss_sub_r

    def forward(self, triplets, s_hist, o_hist, graph_dict, subject=True):
        """model.py:64-104.  With dropout > 0 in training the three dropout sites of the reference are active: the self-loop
        message of both RGCN layers (RGCN.py:36-37), the GRU inputs (Aggregator.py:157-158, inside the fused GRU path with
        Philox masks) and the decoder inputs (model.py:90,99)."""
        return self.decode_loss(*self.encode(triplets, s_hist, o_hist, graph_dict, subject))

    def forward_unfused(self, triplets, s_hist, o_hist, graph_dict, subject=True):
        """Literal model.py:64-104 flow: aggregator -> PackedSequence -> nn.GRU modules (cuDNN).  An API-compatibility /
        cross-check path only; ``forward`` never routes here."""
        if subject:
            rel_embeds = self.rel_embeds[:self.num_rels]
            s, r, o = triplets[:, 0], triplets[:, 1], triplets[:, 2]
            hist, reverse = s_hist, False
        else:
            rel_embeds = self.rel_embeds[self.num_rels:]
            o, r, s = triplets[:, 0], triplets[:, 1], triplets[:, 2]
            hist, reverse = o_hist, True
        p4, p3, hb = self.aggregator._packed(hist, s, r, self.ent_embeds, rel_embeds, graph_dict,
                                             self.global_emb, reverse, True)
        idx = torch.from_numpy(hb.s_idx).to(triplets.device)
        _, s_h = self.encoder(p4)
        s_h = s_h.view(-1, self.h_dim)
        _, s_q = self.encoder_r(p3)
        s_q = s_q.view(-1, self.h_dim)
        pad = torch.zeros(len(s) - s_h.shape[0], self.h_dim, device=s_h.device)
        return self.decode_loss(s[idx], r[idx], o[idx], torch.cat((s_h, pad), 0), torch.cat((s_q, pad), 0),
                                rel_embeds)
