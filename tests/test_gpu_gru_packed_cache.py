"""-m gpu: the packed-weight cache never serves a stale image to the GRU's FFMA fallback.

At h = 8 (3h is not a multiple of 200) renet_gru_fwd packs transposed copies of the weights into its workspace (Brow, Bent,
Brel, Bglob, Whh) and multiplies them with sgemm_nn, which takes the tensor-core engine where the shape allows.  Inside a
weight generation (RGCNAggregator.encode declares one) that engine caches packed B images by B's address.  The workspace
copies are not weights: a later call whose workspace sits elsewhere can hold a different block at an address cached
earlier, and was then served that block's image.  Of this batch's products, H2 @ Brow (S rows) and glob @ Bglob (T rows)
take the tensor-core engine with the same (ldb, N, K); Bglob sits 15 h^2 floats after Brow.  The workspace moves by that
much per call, so each call's Brow lies where the previous call's Bglob did, and every call must equal the uncached
result bit for bit."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import eval_setup, load_npz
from test_forecast_observed_host import _queries

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _operands():
    """The GRU inputs of one batched encode of the golden's subject-side queries (tiny model, h = 8)."""
    from renet_b200 import synthetic
    from renet_b200.inference import _chunk_view
    from renet_b200.utils import global_rows_of_batch
    ctx = eval_setup(DEV)
    m, quads = ctx['model'], ctx['quads']
    ctx['gold'] = load_npz('renet_eval_observed.npz')
    gd, ge = synthetic.build_graph_dict(quads, ctx['dims'][1]), dict(m.global_emb)
    q, hist = _queries(ctx, True)
    (hl, ht, hid, ent_of), has = m._observed_histories(q[:, 0], hist, 'history', gd, ge)
    q_h = np.unique(hid[has])
    view, gs = _chunk_view(hl, ht, q_h, ent_of[q_h], gd)
    s = torch.from_numpy(ent_of[q_h]).to(DEV)
    agg = m.aggregator
    with torch.no_grad():
        hb = agg._batch(view, s, gs, DEV, True)
        H2, readout = agg.aggregate(hb, m.ent_embeds, False)
        glob = global_rows_of_batch(ge, hb, m.h_dim, DEV)
        _, _, seq_s, seq_r = agg._sorted_ids(hb, s, torch.zeros_like(s), DEV)
    return m, hb, H2.contiguous(), readout, glob.contiguous(), seq_s, seq_r


def _gru(ops, ws, nbytes):
    """renet_gru_fwd with the workspace ``ws``: (hn4 | hn3) [Q, 2h]."""
    from renet_b200 import _lib
    from renet_b200.gru import _gru_params
    L, P = _lib.lib(), _lib.ptr
    m, hb, H2, readout, glob, seq_s, seq_r = ops
    h, Q = m.h_dim, hb.num_seq
    p4, p3 = _gru_params(m.encoder), _gru_params(m.encoder_r)
    hn4, hn3 = torch.zeros(Q, h, device=DEV), torch.zeros(Q, h, device=DEV)
    bs = hb.batch_sizes
    rc = L.renet_gru_fwd(P(H2), P(readout), P(hb.row_glob), P(glob), P(m.ent_embeds), P(m.rel_embeds[:m.num_rels]), P(seq_s),
                         P(seq_r), P(hb.graph.seq_len_dev), P(hb.seq_start), bs.ctypes.data_as(ctypes.c_void_p), len(bs),
                         *(P(t) for t in p4), *(P(t) for t in p3), P(hn4), P(hn3), hb.S, Q, glob.shape[0], h, P(ws), nbytes,
                         _lib.stream())
    _lib.check(rc, 'renet_gru_fwd')
    return torch.cat((hn4, hn3), dim=1)


def test_gru_fallback_never_reads_a_stale_packed_image():
    from renet_b200 import _lib
    ops = _operands()
    m, hb = ops[0], ops[1]
    h = m.h_dim
    T = ops[4].shape[0]
    # the FFMA fallback, with both products' row counts at or above the tensor-core engine's minimum of 64
    assert (3 * h) % 200 != 0 and hb.S >= 64 and T >= 64
    nbytes = int(_lib.lib().renet_gru_workspace_bytes(hb.S, hb.num_seq, T, h))
    block = 15 * h * h                                 # floats from Brow to Bglob (Brow, Bent: 6h^2 each; Brel: 3h^2)
    calls = 4
    big = torch.empty(nbytes // 4 + 4 + block * calls, device=DEV)
    with torch.no_grad():
        ref = _gru(ops, big, nbytes)                   # no weight generation: the cache is off
        weights = [m.encoder.weight_ih_l0, m.encoder.weight_hh_l0, m.encoder_r.weight_ih_l0, m.encoder_r.weight_hh_l0]
        with _lib.weight_generation(_lib.new_pack_token(), weights):
            for j in range(calls):
                got = _gru(ops, big[j * block:], nbytes)
                assert torch.equal(got, ref), (j, float((got - ref).abs().max()))
    assert float(ref.abs().max()) > 0
