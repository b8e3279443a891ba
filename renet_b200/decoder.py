"""Fused decoder: linear + cross-entropy of reference model.py:89-91 / 97-100 on the wgmma 3xTF32 engine
(renet_decoder_ce_fwd / _bwd): ``decoder_cross_entropy(x, weight, bias, target)`` equals
``F.cross_entropy(F.linear(x, weight, bias), target)`` (mean over rows) without materialising the [B, |E|] logits in
the forward pass.  ``nn.Linear`` modules stay the parameter holders (state_dict keys ``linear.*`` / ``linear_r.*``).

``decoder_soft_cross_entropy(x, weight, bias, soft_targets)`` is the global model's loss head on the same engine
(renet_decoder_soft_ce_fwd / _bwd): the reference's ``soft_cross_entropy(F.linear(x, weight, bias), soft_targets)``
(utils.py:287-290, fp64 log-softmax, mean over rows), returned as a float64 scalar like the reference's.

``decoder_group_topk(x, weight, bias, row_weight, R, k)`` is the test-time roll-over's candidate scoring on the same engine
(renet_decoder_group_topk): per group of R rows, the k largest row_weight * softmax(F.linear(x, weight, bias)) entries."""
import torch

from . import _lib


class _DecoderCEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, target):
        L, P = _lib.lib(), _lib.ptr
        _lib.require_cuda(x, weight, bias, target)
        x, weight, bias = x.contiguous(), weight.contiguous(), bias.contiguous()
        tgt = target.to(torch.int32).contiguous()
        M, K = x.shape
        N = weight.shape[0]
        dev = x.device
        loss_rows = torch.empty(M, device=dev)
        lse = torch.empty(M, device=dev)
        nbytes = int(L.renet_decoder_ce_workspace_bytes(M, N, K))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _lib.check(L.renet_decoder_ce_fwd(P(x), P(weight), P(bias), P(tgt), P(loss_rows), P(lse), M, N, K, P(ws), nbytes,
                                          _lib.stream()), 'renet_decoder_ce_fwd')
        ctx.save_for_backward(x, weight, bias, tgt, lse)
        return loss_rows.mean()

    @staticmethod
    def backward(ctx, g):
        L, P = _lib.lib(), _lib.ptr
        x, weight, bias, tgt, lse = ctx.saved_tensors
        M, K = x.shape
        N = weight.shape[0]
        dev = x.device
        dx = torch.empty_like(x)
        dw = torch.zeros_like(weight)
        db = torch.zeros_like(bias)
        nbytes = int(L.renet_decoder_ce_bwd_workspace_bytes(M, N, K))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        g = g.contiguous().to(torch.float32)      # the upstream gradient stays on the device (no host read in backward)
        _lib.check(L.renet_decoder_ce_bwd(P(x), P(weight), P(bias), P(tgt), P(lse), 1.0 / M, P(g), P(dx), P(dw), P(db), M, N, K, P(ws),
                                          nbytes, _lib.stream()), 'renet_decoder_ce_bwd')
        return dx, dw, db, None


def decoder_cross_entropy(x, weight, bias, target):
    return _DecoderCEFn.apply(x, weight, bias, target)


class _DecoderSoftCEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, soft_targets):
        L, P = _lib.lib(), _lib.ptr
        _lib.require_cuda(x, weight, bias, soft_targets)
        x, weight, bias = x.contiguous(), weight.contiguous(), bias.contiguous()
        tp = soft_targets.to(torch.float32).contiguous()          # the reference's fp64 targets, converted once
        M, K = x.shape
        N = weight.shape[0]
        dev = x.device
        loss_rows = torch.empty(M, device=dev)
        lse = torch.empty(M, device=dev)
        psum = torch.empty(M, device=dev)
        nbytes = int(L.renet_decoder_soft_ce_workspace_bytes(M, N, K))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _lib.check(L.renet_decoder_soft_ce_fwd(P(x), P(weight), P(bias), P(tp), N, P(loss_rows), P(lse), P(psum), M, N, K, P(ws),
                                               nbytes, _lib.stream()), 'renet_decoder_soft_ce_fwd')
        ctx.save_for_backward(x, weight, bias, tp, lse, psum)
        return loss_rows.double().mean()

    @staticmethod
    def backward(ctx, g):
        L, P = _lib.lib(), _lib.ptr
        x, weight, bias, tp, lse, psum = ctx.saved_tensors
        M, K = x.shape
        N = weight.shape[0]
        dev = x.device
        dx = torch.empty_like(x)
        dw = torch.zeros_like(weight)
        db = torch.zeros_like(bias)
        nbytes = int(L.renet_decoder_soft_ce_bwd_workspace_bytes(M, N, K))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        g = g.contiguous().to(torch.float32)      # the upstream gradient stays on the device (no host read in backward)
        _lib.check(L.renet_decoder_soft_ce_bwd(P(x), P(weight), P(bias), P(tp), N, P(lse), P(psum), 1.0 / M, P(g), P(dx), P(dw),
                                               P(db), M, N, K, P(ws), nbytes, _lib.stream()), 'renet_decoder_soft_ce_bwd')
        return dx, dw, db, None


def decoder_soft_cross_entropy(x, weight, bias, soft_targets):
    return _DecoderSoftCEFn.apply(x, weight, bias, soft_targets)


ORDER_INDEX, ORDER_VALUE = 0, 1          # RENET_TOPK_ORDER_INDEX / RENET_TOPK_ORDER_VALUE
TOPK_MAX_K = 16384                       # RENET_TOPK_MAX_K


def group_topk_capacity(k, size):
    """First candidate-buffer size per group: a few times k covers the entries at or above the threshold in practice; a
    call that needs more says so and is repeated with the exact size."""
    return int(min(size, 4 * k + 256))


def decoder_group_topk(x, weight, bias, row_weight, R, k, order=ORDER_INDEX, capacity=None):
    """renet_decoder_group_topk: the rows of x [G*R, K] in groups of R, p[m, n] = row_weight[m] * softmax(x @ weight^T +
    bias)[m, n]; per group the k largest p and their flat indices r * N + n (ties to the lower index), laid out in
    ``order``.  Returns (values float32 [G, k], indices int64 [G, k]).  ``capacity``: the first candidate-buffer size (a
    group that finds more candidates makes the call run once more with the size it reported)."""
    L, P = _lib.lib(), _lib.ptr
    _lib.require_cuda(x, weight, bias, row_weight)
    x, weight = x.contiguous(), weight.contiguous()
    bias = bias.contiguous() if bias is not None else None
    row_weight = row_weight.to(torch.float32).contiguous()
    M, K = x.shape
    N = weight.shape[0]
    if M % R != 0 or row_weight.numel() != M:
        raise ValueError('decoder_group_topk: %d rows do not form groups of R = %d with one weight each' % (M, R))
    G = M // R
    dev = x.device
    values = torch.empty(G, k, device=dev)
    indices = torch.empty(G, k, dtype=torch.int32, device=dev)
    needed = torch.zeros(1, dtype=torch.int32, device=dev)
    cap = int(capacity) if capacity is not None else group_topk_capacity(k, R * N)
    cap = max(cap, k)
    while True:
        nbytes = int(L.renet_decoder_group_topk_workspace_bytes(G, R, N, K, cap))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _lib.check(L.renet_decoder_group_topk(P(x), P(weight), P(bias), P(row_weight), G, R, N, K, k, order, cap, P(values),
                                              P(indices), P(needed), P(ws), nbytes, _lib.stream()), 'renet_decoder_group_topk')
        need = int(needed.item())
        if need == 0:
            return values, indices.long()
        cap = need
