"""Backward of the fused read-out + GRU through renet_gru_bwd (autograd of Aggregator.py:139-165 +
model.py:86,94)."""
import torch

from . import _lib


def fused_gru_backward(ctx, dhn4, dhn3):
    L = _lib.lib()
    (H2, ent, rel, glob, w_ih4, w_hh4, b_ih4, b_hh4, w_ih3, w_hh3, b_ih3, b_hh3, ws) = ctx.saved_tensors
    hb, seq_s, seq_r = ctx.hb, ctx.seq_s, ctx.seq_r
    h = H2.shape[1]
    S, Q, T, N = hb.S, hb.num_seq, glob.shape[0], H2.shape[0]
    dev = H2.device
    dhn4, dhn3 = dhn4.contiguous(), dhn3.contiguous()
    dH2 = torch.empty_like(H2)
    z = torch.zeros_like
    d_ent, d_rel = z(ent), z(rel)
    d_glob = z(glob) if ctx.needs_input_grad[3] else None
    grads = [z(w_ih4), z(w_hh4), z(b_ih4), z(b_hh4), z(w_ih3), z(w_hh3), z(b_ih3), z(b_hh3)]
    bs = hb.batch_sizes
    if ctx.p_drop > 0.0:
        nbytes = int(L.renet_gru_bwd_dropout_workspace_bytes_len(S, Q, T, h, len(bs)))
        bws = torch.empty(nbytes // 4 + 32, dtype=torch.float32, device=dev)
        dH2.zero_()                                          # the scatter of the masked input gradients accumulates
        rc = L.renet_gru_bwd_dropout(_lib.ptr(H2), _lib.ptr(ctx.readout), _lib.ptr(hb.row_glob), _lib.ptr(glob), _lib.ptr(ent),
                                     _lib.ptr(rel), _lib.ptr(hb.row_seq), _lib.ptr(seq_s), _lib.ptr(seq_r),
                                     _lib.ptr(hb.graph.seq_len_dev), _lib.ptr(hb.seq_start),
                                     bs.ctypes.data_as(_lib.ctypes.c_void_p), len(bs), _lib.ptr(w_ih4), _lib.ptr(w_hh4),
                                     _lib.ptr(w_ih3), _lib.ptr(w_hh3), _lib.ptr(dhn4), _lib.ptr(dhn3), _lib.ptr(dH2),
                                     _lib.ptr(d_ent), _lib.ptr(d_rel), _lib.ptr(d_glob), *[_lib.ptr(g) for g in grads], N, S, Q, T,
                                     h, ctx.p_drop, ctx.seed, _lib.ptr(ws), _lib.ptr(bws), nbytes, _lib.stream())
        _lib.check(rc, 'renet_gru_bwd_dropout')
        return (dH2, d_ent, d_rel, d_glob, *grads, None, None, None, None, None, None)
    nbytes = int(L.renet_gru_bwd_workspace_bytes_len(S, Q, T, h, len(bs)))
    bws = torch.empty(nbytes // 4 + 4, dtype=torch.float32, device=dev)
    rc = L.renet_gru_bwd(_lib.ptr(H2), _lib.ptr(ctx.readout), _lib.ptr(hb.row_glob), _lib.ptr(glob), _lib.ptr(ent),
                         _lib.ptr(rel), _lib.ptr(seq_s), _lib.ptr(seq_r), _lib.ptr(hb.graph.seq_len_dev),
                         _lib.ptr(hb.seq_start), bs.ctypes.data_as(_lib.ctypes.c_void_p), len(bs),
                         _lib.ptr(w_ih4), _lib.ptr(w_hh4), _lib.ptr(w_ih3), _lib.ptr(w_hh3),
                         _lib.ptr(dhn4), _lib.ptr(dhn3), _lib.ptr(dH2), _lib.ptr(d_ent), _lib.ptr(d_rel),
                         _lib.ptr(d_glob), *[_lib.ptr(g) for g in grads], N, S, Q, T, h, _lib.ptr(ws),
                         _lib.ptr(bws), nbytes, _lib.stream())
    _lib.check(rc, 'renet_gru_bwd')
    return (dH2, d_ent, d_rel, d_glob, *grads, None, None, None, None, None, None)
