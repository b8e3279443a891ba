"""Fused decoder: linear + cross-entropy of reference model.py:89-91 / 97-100 on the wgmma 3xTF32 engine
(renet_decoder_ce_fwd / _bwd): ``decoder_cross_entropy(x, weight, bias, target)`` equals
``F.cross_entropy(F.linear(x, weight, bias), target)`` (mean over rows) without materialising the [B, |E|] logits in
the forward pass.  ``nn.Linear`` modules stay the parameter holders (state_dict keys ``linear.*`` / ``linear_r.*``)."""
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
