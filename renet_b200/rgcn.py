"""RGCN layers with the reference's class surface (reference RGCN.py:5-94) on the sm_90a kernels.

``RGCNBlockLayer(in_feat, out_feat, num_rels, num_bases, bias=None, activation=None,
self_loop=False, dropout=0.0)`` keeps the constructor, parameter names/shapes (``weight``
[num_rels, nb*si*so], ``loop_weight`` [in, out]) and ``forward(g, reverse) -> g`` (mutating
``g.ndata['h']``) of the reference, so checkpoints and call sites carry over.  The arithmetic runs in
librenet_b200.so: one self-loop GEMM + one fused gather/transform/reduce/normalise/activation
kernel per layer; backward through the matching CUDA kernels.  There is no PyTorch fallback.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib



def _buf(shape, like, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device=like.device)


class _SelfLoopFn(torch.autograd.Function):
    """loop = Hin @ Wloop with Hin = H[h_index]  (RGCN.py:35 + utils.py:239)."""

    @staticmethod
    def forward(ctx, H, Wloop, h_index, n_rows):
        L = _lib.lib()
        _lib.require_cuda(H, Wloop)
        H, Wloop = H.contiguous(), Wloop.contiguous()
        out = _buf((n_rows, Wloop.shape[1]), H)
        rc = L.renet_selfloop_gemm(_lib.ptr(H), _lib.ptr(h_index), _lib.ptr(Wloop), _lib.ptr(out), n_rows,
                                   H.shape[1], Wloop.shape[1], _lib.stream())
        _lib.check(rc, 'renet_selfloop_gemm')
        ctx.save_for_backward(H, Wloop)
        ctx.h_index, ctx.n_rows = h_index, n_rows
        return out

    @staticmethod
    def backward(ctx, dloop):
        L = _lib.lib()
        H, Wloop = ctx.saved_tensors
        d_in, d_out = Wloop.shape
        dloop = dloop.contiguous()
        dHrows = _buf((ctx.n_rows, d_in), H)
        dWloop = torch.zeros_like(Wloop)
        ws = _buf((d_in * d_out,), H)
        rc = L.renet_selfloop_gemm_bwd(_lib.ptr(H), _lib.ptr(ctx.h_index), _lib.ptr(Wloop), _lib.ptr(dloop),
                                       _lib.ptr(dHrows), _lib.ptr(dWloop), _lib.ptr(ws), ctx.n_rows, d_in, d_out,
                                       _lib.stream())
        _lib.check(rc, 'renet_selfloop_gemm_bwd')
        return _rows_to_table_grad(dHrows, ctx.h_index, H), dWloop, None, None


def _rows_to_table_grad(dHrows, h_index, H):
    """gradient w.r.t. the feature table: identity when not indexed, scatter-add of rows otherwise."""
    if h_index is None:
        return dHrows
    L = _lib.lib()
    dH = torch.zeros_like(H)
    rc = L.renet_scatter_add_rows(_lib.ptr(dHrows), _lib.ptr(h_index), _lib.ptr(dH), dHrows.shape[0],
                                  dHrows.shape[1], _lib.stream())
    _lib.check(rc, 'renet_scatter_add_rows')
    return dH


class _GatherFn(torch.autograd.Function):
    """out = act(norm * sum_e blockdiag(W[type_e]) Hin[src_e] + loop)   (RGCN.py:79-94, 45-48).

    ``loop`` (or None) is consumed in place: the kernel reads it from and writes the result to the same
    buffer."""

    @staticmethod
    def forward(ctx, H, W, loop, h_index, g, reverse, relu, num_bases, d_out):
        L = _lib.lib()
        _lib.require_cuda(H, W)
        H, W = H.contiguous(), W.contiguous()
        if loop is None:
            out = _buf((g.N, d_out), H)
        else:
            out = loop if loop.is_contiguous() else loop.contiguous()
            if out is loop:
                ctx.mark_dirty(loop)
        d_in = H.shape[1]
        hot = g.hot_rel(reverse)       # the dataset's relation ranking when the graph came from a GraphStore
        rc = L.renet_rgcn_gather_hot(_lib.ptr(H), _lib.ptr(h_index), _lib.ptr(W), _lib.ptr(g.row_ptr),
                                     _lib.ptr(g.col_src), _lib.ptr(g.col_type(reverse)), _lib.ptr(g.norm),
                                     _lib.ptr(out), g.N, g.E_launch, d_in, d_out, num_bases, W.shape[0], int(relu),
                                     int(loop is not None), _lib.ptr(hot), 0 if hot is None else hot.numel(), _lib.stream())
        _lib.check(rc, 'renet_rgcn_gather_hot')
        ctx.save_for_backward(H, W, out)
        ctx.g, ctx.reverse, ctx.relu, ctx.nb, ctx.h_index, ctx.has_loop = g, reverse, relu, num_bases, h_index, loop is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        L = _lib.lib()
        H, W, out = ctx.saved_tensors
        g = ctx.g
        d_in, d_out = H.shape[1], out.shape[1]
        dout = dout.contiguous()
        t_row_ptr, t_col_dst, t_col_type, rel_ptr, rel_src, rel_dst = g.backward_structs(ctx.reverse, W.shape[0])
        n_src = getattr(g, 'N_src', g.N)
        dHrows = _buf((n_src, d_in), H)
        dW = torch.zeros_like(W)
        ws = _buf((((g.N * d_out + 3) // 4) * 4 + d_in * d_out,), H)
        if n_src != g.N or hasattr(g, 'N_src'):
            # read-out sub-graph (layer 2): compact destinations, full-graph sources
            rc = L.renet_rgcn_bipartite_bwd(_lib.ptr(H), _lib.ptr(W), _lib.ptr(t_row_ptr), _lib.ptr(t_col_dst),
                                            _lib.ptr(t_col_type), _lib.ptr(rel_ptr), _lib.ptr(rel_src), _lib.ptr(rel_dst),
                                            _lib.ptr(g.norm), _lib.ptr(out), _lib.ptr(dout), _lib.ptr(dHrows), _lib.ptr(dW),
                                            _lib.ptr(ws), n_src, g.N, g.E, d_in, d_out, ctx.nb, W.shape[0], int(ctx.relu),
                                            _lib.stream())
            _lib.check(rc, 'renet_rgcn_bipartite_bwd')
        else:
            rc = L.renet_rgcn_block_bwd(_lib.ptr(H), _lib.ptr(ctx.h_index), _lib.ptr(W), None, _lib.ptr(t_row_ptr),
                                        _lib.ptr(t_col_dst), _lib.ptr(t_col_type), _lib.ptr(rel_ptr),
                                        _lib.ptr(rel_src), _lib.ptr(rel_dst), _lib.ptr(g.norm), _lib.ptr(out),
                                        _lib.ptr(dout), _lib.ptr(dHrows), _lib.ptr(dW), None, _lib.ptr(ws), g.N, g.E,
                                        d_in, d_out, ctx.nb, W.shape[0], int(ctx.relu), _lib.stream())
            _lib.check(rc, 'renet_rgcn_block_bwd')
        dloop = ws[:g.N * d_out].view(g.N, d_out) if ctx.has_loop else None     # P = dout * act'(out)
        return _rows_to_table_grad(dHrows, ctx.h_index, H), dW, dloop, None, None, None, None, None, None


class RGCNLayer(nn.Module):
    """Reference RGCN.py:5-51 (constructor and attributes kept)."""

    def __init__(self, in_feat, out_feat, bias=None, activation=None, self_loop=False, dropout=0.0):
        super(RGCNLayer, self).__init__()
        self.bias = bias
        self.activation = activation
        self.self_loop = self_loop
        if self.bias == True:  # noqa: E712 - the reference compares with == True (RGCN.py:13)
            # reference RGCN.py:14-16 calls xavier_uniform_ on a 1-D tensor, which raises; bias=True
            # is never used by RE-Net.  Zero-initialised here.
            self.bias = nn.Parameter(torch.zeros(out_feat))
        if self.self_loop:
            self.loop_weight = nn.Parameter(torch.Tensor(in_feat, out_feat))
            nn.init.xavier_uniform_(self.loop_weight, gain=nn.init.calculate_gain('relu'))
        self.dropout = nn.Dropout(dropout) if dropout else None

    def propagate(self, g, reverse):
        raise NotImplementedError

    def forward(self, g, reverse):
        raise NotImplementedError


class RGCNBlockLayer(RGCNLayer):
    """Reference RGCN.py:54-94: block-diagonal-decomposed relational graph convolution."""

    def __init__(self, in_feat, out_feat, num_rels, num_bases, bias=None, activation=None, self_loop=False,
                 dropout=0.0):
        super(RGCNBlockLayer, self).__init__(in_feat, out_feat, bias, activation, self_loop=self_loop,
                                             dropout=dropout)
        self.num_rels = num_rels
        self.num_bases = num_bases
        assert self.num_bases > 0
        self.out_feat = out_feat
        self.submat_in = in_feat // self.num_bases
        self.submat_out = out_feat // self.num_bases
        self.weight = nn.Parameter(torch.Tensor(self.num_rels, self.num_bases * self.submat_in * self.submat_out))
        nn.init.xavier_uniform_(self.weight, gain=nn.init.calculate_gain('relu'))

    def _relu_fused(self):
        return self.activation is F.relu or self.activation is torch.relu

    def forward(self, g, reverse):
        """g: BatchedHistoryGraph.  Reads g.ndata['h'] (or the virtual ent_embeds[id] view), writes the
        layer output back to g.ndata['h'] and returns g, like reference RGCN.py:33-51."""
        if g.h_table is not None and 'h' not in g.ndata:
            H, h_index = g.h_table, g.h_index
        else:
            H, h_index = g.ndata['h'], None
        out = self.apply_layer(g, H, h_index, reverse)
        g.ndata['h'] = out
        g.h_table = g.h_index = None
        return g

    def apply_layer(self, g, H, h_index, reverse, loop_index=None):
        """One layer over graph ``g``.  ``h_index``: rows of H are addressed through it (fused embedding lookup);
        ``loop_index`` (read-out sub-graph): destination u's own feature row is H[loop_index[u]] while edge sources
        address H directly."""
        if isinstance(self.bias, nn.Parameter):                 # RGCN.py:43-44 (never used by RE-Net)
            raise RuntimeError('RGCNBlockLayer(bias=True) is not supported by the fused kernel')
        loop = None
        if self.self_loop:
            loop = _SelfLoopFn.apply(H, self.loop_weight, h_index if loop_index is None else loop_index, g.N)
            if self.dropout is not None:
                loop = self.dropout(loop)                       # RGCN.py:36-37
        fuse_relu = self._relu_fused()
        out = _GatherFn.apply(H, self.weight, loop, h_index, g, reverse, fuse_relu, self.num_bases, self.out_feat)
        if self.activation is not None and not fuse_relu:
            out = self.activation(out)
        return out

    def propagate(self, g, reverse):
        """Reference RGCN.py:90-91 (message passing only, no self-loop / activation)."""
        H = g.ndata['h']
        g.h_table = g.h_index = None
        g.ndata['h'] = _GatherFn.apply(H, self.weight, None, None, g, reverse, False, self.num_bases, self.out_feat)
