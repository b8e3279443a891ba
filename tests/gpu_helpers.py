"""Helpers for the -m gpu parity tests: everything goes through the C-ABI (renet_b200._lib)."""
import numpy as np
import torch

from renet_b200 import _lib
from renet_b200.graph import build_csr

DEV = 'cuda:0'


def d(x, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(x))
    if dtype is not None:
        t = t.to(dtype)
    return t.to(DEV)


def coo_to_csr(src, dst, etype, N):
    """device CSR by destination via renet_build_csr -> (row_ptr, col_src, col_type)"""
    rp, cs, ct, _ = build_csr(d(dst, torch.int32), d(src, torch.int32), d(etype, torch.int32), N)
    return rp, cs, ct


def layer_fwd(H, h_index, W, Wloop, rp, cs, ct, norm, N, E, d_in, d_out, nb, relu):
    L = _lib.lib()
    out = torch.empty(N, d_out, device=DEV)
    rc = L.renet_rgcn_block_fwd(_lib.ptr(H), _lib.ptr(h_index), _lib.ptr(W), _lib.ptr(Wloop), _lib.ptr(rp),
                                _lib.ptr(cs), _lib.ptr(ct), _lib.ptr(norm), _lib.ptr(out), N, E, d_in, d_out, nb,
                                W.shape[0], int(relu), _lib.stream())
    _lib.check(rc, 'renet_rgcn_block_fwd')
    return out


def layer_bwd(H, h_index, W, Wloop, src, dst, etype, norm, out, dout, N, E, d_in, d_out, nb, relu):
    """builds the backward edge structures with renet_build_csr and calls renet_rgcn_block_bwd.  dW and dWloop are
    accumulated (+=): they start from a random non-zero base, and what is returned is the result minus that base (in
    float64), so a kernel that overwrote or misread the base fails the comparison with the reference gradient."""
    L = _lib.lib()
    R2 = W.shape[0]
    s32, d32, t32 = d(src, torch.int32), d(dst, torch.int32), d(etype, torch.int32)
    t_rp, t_cd, t_ct, _ = build_csr(s32, d32, t32, N)               # keyed by source
    r_rp, r_src, r_dst, _ = build_csr(t32, s32, d32, R2)             # keyed by relation
    dH = torch.empty(N, d_in, device=DEV)
    # 1e-2: far above the 1e-4 bar relative to these gradients if it were lost, small enough that rounding base + gradient
    # to fp32 stays far below it
    gen = torch.Generator(device=DEV).manual_seed(N + E)
    dW = torch.randn(W.shape, device=DEV, generator=gen) * 1e-2
    dWl = torch.randn(Wloop.shape, device=DEV, generator=gen) * 1e-2 if Wloop is not None else None
    base_W, base_Wl = dW.clone(), (dWl.clone() if dWl is not None else None)
    ws = torch.empty(((N * d_out + 3) // 4) * 4 + d_in * d_out, device=DEV)
    rc = L.renet_rgcn_block_bwd(_lib.ptr(H), _lib.ptr(h_index), _lib.ptr(W), _lib.ptr(Wloop), _lib.ptr(t_rp),
                                _lib.ptr(t_cd), _lib.ptr(t_ct), _lib.ptr(r_rp), _lib.ptr(r_src), _lib.ptr(r_dst),
                                _lib.ptr(norm), _lib.ptr(out), _lib.ptr(dout), _lib.ptr(dH), _lib.ptr(dW),
                                _lib.ptr(dWl), _lib.ptr(ws), N, E, d_in, d_out, nb, R2, int(relu), _lib.stream())
    _lib.check(rc, 'renet_rgcn_block_bwd')
    return dH, dW.double() - base_W.double(), (dWl.double() - base_Wl.double() if dWl is not None else None)
