"""Fused read-out + concat + GRU (reference Aggregator.py:139-165 + model.py:86,94) via renet_gru_fwd.

``fused_gru`` consumes the layer-2 node features, the embedding tables and the two ``nn.GRU`` modules'
own parameters (so state_dict keys ``encoder.*`` / ``encoder_r.*`` are the reference's) and returns
the final hidden state of both encoders for the non-empty sequences, sorted as the reference sorts
them (by history length, descending).
"""
import torch

from . import _lib


def _gru_params(m):
    if m.num_layers != 1 or m.bidirectional or not m.bias:
        raise RuntimeError('renet_b200 fused GRU supports the reference configuration only '
                           '(1 layer, unidirectional, with bias; model.py:28-29)')
    return m.weight_ih_l0, m.weight_hh_l0, m.bias_ih_l0, m.bias_hh_l0


class _FusedGruFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, H2, ent, rel, glob, w_ih4, w_hh4, b_ih4, b_hh4, w_ih3, w_hh3, b_ih3, b_hh3, hb, seq_s, seq_r, readout=None,
                p_drop=0.0, seed=0):
        L = _lib.lib()
        tensors = [t.contiguous() for t in (H2, ent, rel, glob, w_ih4, w_hh4, b_ih4, b_hh4, w_ih3, w_hh3, b_ih3, b_hh3)]
        _lib.require_cuda(*tensors)
        H2, ent, rel, glob, w_ih4, w_hh4, b_ih4, b_hh4, w_ih3, w_hh3, b_ih3, b_hh3 = tensors
        h = H2.shape[1]
        S, Q, T = hb.S, hb.num_seq, glob.shape[0]
        dev = H2.device
        hn4 = torch.zeros(Q, h, device=dev)
        hn3 = torch.zeros(Q, h, device=dev)
        readout = hb.readout if readout is None else readout
        bs = hb.batch_sizes      # host int32 numpy
        if p_drop > 0.0:
            # training with input dropout (Aggregator.py:157-158): masked inputs materialised in the workspace, Philox masks
            nbytes = int(L.renet_gru_dropout_workspace_bytes_len(S, Q, T, h, len(bs)))
            ws = torch.empty(nbytes // 4 + 32, dtype=torch.float32, device=dev)
            rc = L.renet_gru_fwd_dropout(_lib.ptr(H2), _lib.ptr(readout), _lib.ptr(hb.row_glob), _lib.ptr(glob),
                                         _lib.ptr(ent), _lib.ptr(rel), _lib.ptr(hb.row_seq), _lib.ptr(seq_s), _lib.ptr(seq_r),
                                         _lib.ptr(hb.graph.seq_len_dev), _lib.ptr(hb.seq_start),
                                         bs.ctypes.data_as(_lib.ctypes.c_void_p), len(bs),
                                         _lib.ptr(w_ih4), _lib.ptr(w_hh4), _lib.ptr(b_ih4), _lib.ptr(b_hh4),
                                         _lib.ptr(w_ih3), _lib.ptr(w_hh3), _lib.ptr(b_ih3), _lib.ptr(b_hh3),
                                         _lib.ptr(hn4), _lib.ptr(hn3), S, Q, T, h, float(p_drop), int(seed), _lib.ptr(ws), nbytes,
                                         _lib.stream())
            _lib.check(rc, 'renet_gru_fwd_dropout')
        else:
            nbytes = int(L.renet_gru_workspace_bytes_len(S, Q, T, h, len(bs)))
            ws = torch.empty(nbytes // 4 + 4, dtype=torch.float32, device=dev)
            rc = L.renet_gru_fwd(_lib.ptr(H2), _lib.ptr(readout), _lib.ptr(hb.row_glob), _lib.ptr(glob),
                                 _lib.ptr(ent), _lib.ptr(rel), _lib.ptr(seq_s), _lib.ptr(seq_r),
                                 _lib.ptr(hb.graph.seq_len_dev), _lib.ptr(hb.seq_start),
                                 bs.ctypes.data_as(_lib.ctypes.c_void_p), len(bs),
                                 _lib.ptr(w_ih4), _lib.ptr(w_hh4), _lib.ptr(b_ih4), _lib.ptr(b_hh4),
                                 _lib.ptr(w_ih3), _lib.ptr(w_hh3), _lib.ptr(b_ih3), _lib.ptr(b_hh3),
                                 _lib.ptr(hn4), _lib.ptr(hn3), S, Q, T, h, _lib.ptr(ws), nbytes, _lib.stream())
        _lib.check(rc, 'renet_gru_fwd')
        ctx.save_for_backward(*tensors, ws)
        ctx.hb, ctx.seq_s, ctx.seq_r, ctx.readout, ctx.p_drop, ctx.seed = hb, seq_s, seq_r, readout, float(p_drop), int(seed)
        return hn4, hn3

    @staticmethod
    def backward(ctx, dhn4, dhn3):
        from .gru_bwd import fused_gru_backward
        return fused_gru_backward(ctx, dhn4, dhn3)


def fused_gru(H2, ent, rel, glob, hb, seq_s, seq_r, encoder, encoder_r, readout=None, p_drop=0.0, seed=None):
    """``readout`` overrides hb.readout: rows of H2 the sequences read (the compact indices of the read-out sub-graph).
    ``p_drop`` > 0: input dropout of the reference's aggregator (Aggregator.py:157-158) inside the fused path, masks from
    Philox keyed by ``seed`` (drawn from torch's default CPU generator when not given, so torch.manual_seed makes runs
    repeatable)."""
    p4, p3 = _gru_params(encoder), _gru_params(encoder_r)
    if p_drop > 0.0 and seed is None:
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    return _FusedGruFn.apply(H2, ent, rel, glob, *p4, *p3, hb, seq_s, seq_r, readout, float(p_drop), int(seed or 0))
