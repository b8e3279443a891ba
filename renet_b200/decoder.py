"""Fused decoder: linear + cross-entropy of reference model.py:89-91 / 97-100 on the wgmma 3xTF32 engine
(renet_decoder_ce_fwd / _bwd): ``decoder_cross_entropy(x, weight, bias, target)`` equals
``F.cross_entropy(F.linear(x, weight, bias), target)`` (mean over rows) without materialising the [B, |E|] logits in
the forward pass.  ``nn.Linear`` modules stay the parameter holders (state_dict keys ``linear.*`` / ``linear_r.*``).

``decoder_soft_cross_entropy(x, weight, bias, soft_targets)`` is the global model's loss head on the same engine
(renet_decoder_soft_ce_fwd / _bwd): the reference's ``soft_cross_entropy(F.linear(x, weight, bias), soft_targets)``
(utils.py:287-290, fp64 log-softmax, mean over rows), returned as a float64 scalar like the reference's.

``decoder_group_topk(x, weight, bias, row_weight, R, k)`` is the test-time roll-over's candidate scoring on the same engine
(renet_decoder_group_topk): per group of R rows, the k largest row_weight * softmax(F.linear(x, weight, bias)) entries.

``decoder_rank(x, weight, bias, label, exclude)`` is the test-time scoring on the same engine (renet_decoder_rank): per row
the cross-entropy loss and the label's raw and filtered ranks by the reference's tie rule (model.py:373-379, 403-418).
``decoder_rank_counts_multi(x, weight, bias, label, excludes)`` counts against up to two filters in the same pass
(renet_decoder_rank_multi): the static and the time-aware filter of ``evaluate_stream(time_aware=True)``."""
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


def decoder_rank_counts(x, weight, bias, label, exclude=None):
    """renet_decoder_rank: for z = x @ weight^T + bias and the labels ``label`` [M], returns (loss_rows float32 [M],
    counts int32 [M, 4]) with counts[m] = (#z > z_l, #z == z_l, #p > p_l, #p == p_l) where p = torch.sigmoid(z) with the
    columns of row m's exclusion list other than its label set to 0.  ``exclude`` = (col, begin, end): int32 device
    tensors, row m's list being col[begin[m]:end[m]] in ascending order; None leaves the last two counts 0."""
    L, P = _lib.lib(), _lib.ptr
    _lib.require_cuda(x, weight, label)
    x, weight = x.contiguous(), weight.contiguous()
    bias = bias.contiguous() if bias is not None else None
    lab = label.to(torch.int32).contiguous()
    M, K = x.shape
    N = weight.shape[0]
    if lab.numel() != M:
        raise ValueError('decoder_rank: %d rows but %d labels' % (M, lab.numel()))
    col = begin = end = None
    if exclude is not None:
        col, begin, end = (t.to(torch.int32).contiguous() for t in exclude)
        _lib.require_cuda(col, begin, end)
        if begin.numel() != M or end.numel() != M:
            raise ValueError('decoder_rank: exclusion ranges need one (begin, end) per row')
    dev = x.device
    loss_rows = torch.empty(M, device=dev)
    counts = torch.empty(M, 4, dtype=torch.int32, device=dev)
    nbytes = int(L.renet_decoder_rank_workspace_bytes(M, N, K))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _lib.check(L.renet_decoder_rank(P(x), P(weight), P(bias), P(lab), P(col), P(begin), P(end), P(loss_rows), P(counts), M, N, K,
                                    P(ws), nbytes, _lib.stream()), 'renet_decoder_rank')
    return loss_rows, counts


def decoder_rank_counts_multi(x, weight, bias, label, excludes):
    """renet_decoder_rank_multi: decoder_rank_counts against several filters in one pass.  ``excludes`` is a list of up to
    two (col, begin, end) exclusion lists as in decoder_rank_counts.  Returns (loss_rows float32 [M], counts int32
    [M, 2 + 2L]): counts[m, :2] is the raw pair and counts[m, 2 + 2j : 4 + 2j] the filtered pair against list j, each
    equal to what decoder_rank_counts gives with that list alone."""
    L, P = _lib.lib(), _lib.ptr
    _lib.require_cuda(x, weight, label)
    x, weight = x.contiguous(), weight.contiguous()
    bias = bias.contiguous() if bias is not None else None
    lab = label.to(torch.int32).contiguous()
    M, K = x.shape
    N = weight.shape[0]
    if lab.numel() != M:
        raise ValueError('decoder_rank_counts_multi: %d rows but %d labels' % (M, lab.numel()))
    excludes = list(excludes)
    n = len(excludes)
    if n > 2:
        raise ValueError('decoder_rank_counts_multi: at most two exclusion lists, got %d' % n)
    col = begin = end = None
    if n:
        cols, begins, ends, off = [], [], [], 0
        for ex in excludes:
            c, b, e = (t.to(torch.int32).contiguous() for t in ex)
            _lib.require_cuda(c, b, e)
            if b.numel() != M or e.numel() != M:
                raise ValueError('decoder_rank_counts_multi: exclusion ranges need one (begin, end) per row')
            cols.append(c)
            begins.append(b + off)                   # into the shared column array
            ends.append(e + off)
            off += c.numel()
        col, begin, end = torch.cat(cols), torch.cat(begins), torch.cat(ends)
    dev = x.device
    loss_rows = torch.empty(M, device=dev)
    counts = torch.empty(M, 2 + 2 * n, dtype=torch.int32, device=dev)
    nbytes = int(L.renet_decoder_rank_workspace_bytes(M, N, K))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _lib.check(L.renet_decoder_rank_multi(P(x), P(weight), P(bias), P(lab), n, P(col), P(begin), P(end), P(loss_rows), P(counts),
                                          M, N, K, P(ws), nbytes, _lib.stream()), 'renet_decoder_rank_multi')
    return loss_rows, counts


def ranks_from_counts(greater, equal):
    """The reference's tie rule (model.py:373-379): #greater + (#equal - 1) / 2 + 1, in float64."""
    return greater.double() + (equal.double() - 1.0) / 2 + 1


def decoder_rank(x, weight, bias, label, exclude=None):
    """(loss_rows float32 [M], raw ranks float64 [M], filtered ranks float64 [M] or None when ``exclude`` is None) of the
    labels among the rows of x @ weight^T + bias; see decoder_rank_counts."""
    loss_rows, c = decoder_rank_counts(x, weight, bias, label, exclude)
    raw = ranks_from_counts(c[:, 0], c[:, 1])
    filt = ranks_from_counts(c[:, 2], c[:, 3]) if exclude is not None else None
    return loss_rows, raw, filt
