"""The RE-Net training step (DataParallelTrainer.train_step: RENet.forward for both directions, backward, the native clip +
Adam over the flat buffers) per row against float64 at the datasets' shapes, with dropout on (cases for
tests/test_gpu_step_contract.py; importing this module needs no GPU).

What is checked is how the step is put together: the loss of both directions (decode_loss pairing s[idx], r[idx], o[idx]
with the sorted s_h / s_q rows, the relation loss weighted 0.1, each direction's half of rel_embeds), every parameter's
gradient summed over both directions and all its sources, the dropout masks of every site, the trainer's flat buffers
(reversed order, ALIGN padding, every parameter a view of flat_p) and the clip + Adam step over them, over several steps.
Each kernel family has its own suite.

Reference.  Float64 on the device.  The encoder of each direction is encoder_contract_check.restate_dir with the recorded
masks; the decoder and loss follow model.py:89-103 as oracle/restate.renet_forward restates them, with the recorded
decoder masks; gradients are fp64 autograd of loss_s + loss_o over every parameter.  Layer 1's ReLU derivative is the
kernel's own H1 > 0, recorded from the training forward (a hook on rgcn1.apply_layer's output).  Each step is restated
from the parameters the model holds when the step starts (read back through the model after the previous step).

Masks.  Every nn.Dropout is a global_contract_check.RecordingDropout (keeping .p, which the fused GRU reads): per
direction one mask for rgcn1's self-loop rows [N, h], one for rgcn2's [U, h] (the read-out sub-graph's compact rows, placed
on the nodes sub.uniq names), two for RENet.dropout (x [B, 3h], x_r [B, 2h]) and none for aggregator.dropout (a mask there
would mean the unfused GRU ran).  The fused GRU's masks are regenerated from the Philox seed it is launched with
(recorded from _FusedGruFn.apply; one per direction, the two different): X4's from offset 0, X3's from S * 4h, by
mask_torch, a torch port of support_contract_check.mask_ref that each case checks against mask_ref on a sample.

Bars.  The loss within LOSS_TOL relative.  s_h / s_q and every gradient row as in the encoder suite:
|err|_inf <= tau (|ref_row|_inf + 1e-2 |ref|_inf), tau = 1e-4 (s_h, s_q) / 5e-4 (gradients: each row of ent_embeds,
rel_embeds, the RGCN weights, the loop weights, the GRU matrices and the linear layers, each bias vector as a whole); rows
fp64 leaves at exactly 0 must be exactly 0.  The gradients are read from flat_g by a wrapped optimizer_step before the
native step runs.  Clip + Adam: from that flat_g, the previous flat_p, exp_avg and exp_avg_sq, clip_grad_norm_'s
coefficient max_norm / (|g| + 1e-6) capped at 1 (|g| from the kernel's sum of squares, itself checked against fp64 under
the support suite's bar) and Adam with weight decay in fp64, every element under the support suite's Adam bound.  The
kernel's own gradient is used there, not the fp64 one: Adam's first steps normalise the update, so a gradient difference
within the bar would show as a whole lr.  ALIGN padding stays 0, every named parameter aliases flat_p at the offset the
layout rule gives, step_count advances by 1, and each case asserts its clip regime with a margin of 2x.

Discriminating power.  Before any GPU comparison, each case applies these mistakes to its float64 restatement at its
second step (its first when it has one) and asserts each misses the bar by at least MISS (the largest ratio over the loss,
s_h / s_q rows and gradient rows; over the Adam elements for the last three):
  rel-weight       the relation loss weighted 1.0 instead of 0.1
  dec-rel-half     the object direction's decoder reads the subject half of rel_embeds
  unsorted         the decoder pairs s_h with the unsorted (s, r, o)
  x3-mask          X3 uses X4's mask (offset 0 for both)
  loop2-shift      layer 2's self-loop mask shifted by one read-out node
  shared-mask      the two decoder inputs share one mask
  no-dec-ent-grad  ent_embeds gets no gradient from the decoder
  drop-obj-loss    the object direction's loss is dropped
  stale            the step restated from the previous step's parameters (the symptom of stale packed weights)
  adam-no-wd       Adam without weight decay
  clip-per-dir     the clip coefficient taken per direction
  adam-bias-step   the bias corrections one step off
A mistake a case cannot express (no dropout, one step, no clipping) is n/a there; each case lists what it requires.

Which kernels ran, from torch.profiler (the union over up to ten traces of a further step): with dropout
pack_inputs_dropout_kernel and unpack_inputs_dropout_kernel, or in deterministic mode dropout_grad_rows_kernel and
scatter_add_rows_sorted_kernel; the RGCN forward gather kernel (and the stream kernel's StCfg) each case names for
layers 1 and 2, which must also be what the dispatch rule of rgcn_fwd.cu gives for the recorded sizes; the decoder CE
kernels; no cuDNN RNN kernel."""
import contextlib
import re
import time

import numpy as np
import torch

import encoder_contract_check as enc
import global_contract_check as glb
import support_contract_check as sup

DEV = 'cuda:0'
TAU_FWD, TAU_GRAD = enc.TAU_FWD, enc.TAU_GRAD
LOSS_TOL = 1e-5
MISS = 10.0
P_DROP = 0.5
LR, WD, BETAS, EPS = 1e-3, 1e-5, (0.9, 0.999), 1e-8      # bench.py's train_region
REGIME_MARGIN = 2.0
CLIP_NORM = 0.05           # the cases that clip: about a fifth of the gradient norm of these models' first steps
WORST = {}                 # output -> (largest err / bar, case)
MISSES = {}                # mistake -> (smallest miss / bar over the cases, case)
SECONDS = {}
DEC_MUTS = ('rel-weight', 'dec-rel-half', 'unsorted', 'shared-mask', 'no-dec-ent-grad', 'drop-obj-loss')
ENC_MUTS = ('x3-mask', 'loop2-shift')
ADAM_MUTS = ('adam-no-wd', 'clip-per-dir', 'adam-bias-step')
ALL_MUTS = DEC_MUTS + ENC_MUTS + ('stale',) + ADAM_MUTS
NO_DROPOUT_MUTS = ('rel-weight', 'dec-rel-half', 'unsorted', 'no-dec-ent-grad', 'drop-obj-loss', 'stale') + ADAM_MUTS


# ---- the GRU's Philox masks in torch --------------------------------------------------------------------------------------------
_M32 = 0xFFFFFFFF


def _mulhilo(a, m):
    """(high, low) 32-bit words of a * m, a an int64 tensor of 32-bit values, m a 32-bit constant, without leaving int64"""
    hi_part, lo_part = a * (m >> 16), a * (m & 0xFFFF)          # each < 2^48
    mid = ((hi_part & 0xFFFF) << 16) + lo_part
    return (hi_part >> 16) + (mid >> 32), mid & _M32


def mask_torch(seed, offset, n, p, device=DEV):
    """support_contract_check.mask_ref on a torch device: Philox4x32-10 per counter idx >> 2 (key = seed), word idx & 3"""
    c_lo, c_hi = offset >> 2, (offset + n - 1) >> 2
    ctr = torch.arange(c_lo, c_hi + 1, dtype=torch.int64, device=device)
    zero = torch.zeros_like(ctr)
    c = [ctr & _M32, ctr >> 32, zero, zero]
    k0, k1 = seed & _M32, seed >> 32
    for _ in range(10):
        hi0, lo0 = _mulhilo(c[0], sup.PHILOX_M0)
        hi1, lo1 = _mulhilo(c[2], sup.PHILOX_M1)
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0, k1 = (k0 + sup.PHILOX_W0) & _M32, (k1 + sup.PHILOX_W1) & _M32
    w = torch.stack(c, 1).reshape(-1)[offset - 4 * c_lo:][:n]
    u = w.to(torch.float32) * np.float32(2.0 ** -32)
    keep = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))
    return torch.where(u >= torch.tensor(np.float32(p), device=device), keep, 0.0).to(torch.float32)


def check_mask_port(seed, S, h, p):
    """the port against the numpy restatement on a sample at both masks' starts"""
    for off in (0, S * 4 * h, S * 4 * h - 5):
        n = min(4099, S * 7 * h - off)
        got = mask_torch(seed, off, n, p).cpu().numpy()
        assert np.array_equal(got, sup.mask_ref(seed, off, n, p)), ('mask_torch differs from mask_ref', seed, off)


# ---- the package's step -------------------------------------------------------------------------------------------------------------
def make_model(d, p, seed):
    from renet_b200.model import RENet
    torch.manual_seed(seed)
    m = RENet(d.num_e, d.h, d.R, dropout=p, num_bases=d.nb).to(DEV)
    with torch.no_grad():
        for layer in (m.aggregator.rgcn1, m.aggregator.rgcn2):      # as the encoder suite (make_model there)
            layer.weight.mul_(enc.RGCN_SCALE)
    m.global_emb = d.glob
    return m


@contextlib.contextmanager
def spies(m):
    """records per RGCNAggregator.encode call its s_h, s_q and batch, layer 1's H1 > 0 and graph size, layer 2's loop_index
    (sub.uniq) and graph size, and the fused GRU's dropout probability and Philox seed"""
    from renet_b200 import gru
    rec = {'enc': [], 'l1': [], 'l2': [], 'gru': []}
    agg = m.aggregator
    orig_encode, orig1, orig2, orig_fn = agg.encode, agg.rgcn1.apply_layer, agg.rgcn2.apply_layer, gru._FusedGruFn

    def encode(*a, **k):
        s_h, s_q, hb = orig_encode(*a, **k)
        rec['enc'].append((s_h.detach().clone(), s_q.detach().clone(), hb))
        return s_h, s_q, hb

    def apply1(g, *a, **k):
        E = int(g.E_launch)
        out = orig1(g, *a, **k)
        rec['l1'].append((out.detach() > 0, int(g.N), E))
        return out

    def apply2(g, H, h_index, reverse, loop_index=None):
        rec['l2'].append((loop_index.long().clone(), int(g.N), int(g.E_launch)))
        return orig2(g, H, h_index, reverse, loop_index=loop_index)

    class Fn:
        @staticmethod
        def apply(*a):
            rec['gru'].append((float(a[-2]), int(a[-1])))
            return orig_fn.apply(*a)
    agg.encode, agg.rgcn1.apply_layer, agg.rgcn2.apply_layer, gru._FusedGruFn = encode, apply1, apply2, Fn
    try:
        yield rec
    finally:
        gru._FusedGruFn = orig_fn
        del agg.encode, agg.rgcn1.apply_layer, agg.rgcn2.apply_layer


def layout(m):
    """{name: (offset, numel)} of the flat buffers by the trainer's rule: parameters in reverse registration order, each
    starting on an ALIGN boundary"""
    from renet_b200.parallel import ALIGN
    assert (ALIGN * 4) % 256 == 0
    named = [(k, p) for k, p in m.named_parameters() if p.requires_grad][::-1]
    out, o = {}, 0
    for k, p in named:
        out[k] = (o, p.numel())
        o += -(-p.numel() // ALIGN) * ALIGN
    return out, o


def inputs_of(d, feed):
    """train_step's (s_hist, o_hist, graph_dict) for one batch"""
    if feed == 'lists':
        return d.hist[False], d.hist[True], d.gd_pkg
    vs, gs = d.view(False, hint=False if feed == 'prefetch' else None)
    vo, _ = d.view(True, hint=True if feed == 'prefetch' else None)
    return vs, vo, gs


class StepRec:
    pass


def run_steps(m, tr, batches, feed, cap):
    """train_step over the batches -> [StepRec]: what each step started from, what the kernels computed, the masks"""
    recs = glb.swap_dropouts(m) if not hasattr(m, '_recs') else m._recs
    m._recs = recs
    ins = [inputs_of(d, feed) for d in batches]
    if feed == 'prefetch':
        from renet_b200 import hoststore
        hbs = list(hoststore.prefetch([(a, b) for a, b, _ in ins], DEV))
        ins = [(hs, ho, gd) for (hs, ho), (_, _, gd) in zip(hbs, ins)]
    out = []
    for d, (sh, oh, gd) in zip(batches, ins):
        st = StepRec()
        st.d = d
        st.P = {k: p.detach().clone() for k, p in m.named_parameters()}
        for r in recs.values():
            r.masks.clear()
        n0 = tr.step_count
        with spies(m) as rec:
            st.loss = tr.train_step(torch.from_numpy(d.trip).to(DEV), sh, oh, gd)
        assert tr.step_count == n0 + 1, 'step_count did not advance by 1'
        st.opt = cap.pop()
        assert not cap and st.opt['step'] == n0 + 1
        st.after = {k: getattr(tr, k).clone() for k in ('flat_p', 'exp_avg', 'exp_avg_sq')}
        st.rec, st.masks = rec, {k: list(r.masks) for k, r in recs.items()}
        out.append(st)
    return out


def make_trainer(m, max_norm):
    from renet_b200 import parallel
    cap = []

    def opt(tr):
        c = {'g': tr.flat_g.clone(), 'p': tr.flat_p.clone(), 'm': tr.exp_avg.clone(), 'v': tr.exp_avg_sq.clone(),
             'step': tr.step_count}
        parallel.native_optimizer_step(tr)
        c['sumsq'] = float(tr._sumsq[0])
        cap.append(c)
    tr = parallel.DataParallelTrainer(m, lr=LR, weight_decay=WD, betas=BETAS, eps=EPS, grad_norm=max_norm, optimizer_step=opt)
    return tr, cap


def masks_of(case, st, p):
    """per direction: the restatement's masks (None without dropout) from the recordings of one step"""
    rec, ms = st.rec, st.masks
    assert len(rec['enc']) == 2 and len(rec['l1']) == 2 and len(rec['l2']) == 2 and len(rec['gru']) == 2, (
        case, {k: len(v) for k, v in rec.items()})
    if p:
        assert [len(ms[k]) for k in ('aggregator.rgcn1.dropout', 'aggregator.rgcn2.dropout', 'dropout', 'aggregator.dropout')] \
            == [2, 2, 4, 0], (case, {k: len(v) for k, v in ms.items()})
    else:
        assert all(len(v) == 0 for v in ms.values()), (case, 'a dropout mask at p = 0')
    seeds = [s for _, s in rec['gru']]
    assert all(q == p for q, _ in rec['gru']), (case, 'the fused GRU ran with another p', rec['gru'])
    if p:
        assert seeds[0] != seeds[1], (case, 'both directions drew one Philox seed')
    out = {}
    for rev in (False, True):
        i = int(rev)
        s_h, s_q, hb = rec['enc'][i]
        relu1, N, _ = rec['l1'][i]
        uniq, U_cap, _ = rec['l2'][i]
        dm = {'relu1': relu1, 'hb': hb, 's_h': s_h, 's_q': s_q, 'N': N}
        readout = hb.readout[:hb.S].long()
        U = int(torch.unique(readout).numel())
        assert U_cap == hb.S and torch.equal(uniq[:U], torch.unique(readout)), (case, 'sub.uniq is not the distinct read-out rows')
        dm['uniq'] = uniq[:U]
        if p:
            h = s_h.shape[1]
            dm['loop1'] = ms['aggregator.rgcn1.dropout'][i]
            dm['sub2'] = ms['aggregator.rgcn2.dropout'][i][:U]
            assert dm['loop1'].shape == (N, h) and ms['aggregator.rgcn2.dropout'][i].shape == (hb.S, h), case
            dm['loop2'] = place2(dm['sub2'], dm['uniq'], N)
            check_mask_port(seeds[i], hb.S, h, p)
            dm['x4'] = mask_torch(seeds[i], 0, hb.S * 4 * h, p).view(hb.S, 4 * h)
            dm['x3'] = mask_torch(seeds[i], hb.S * 4 * h, hb.S * 3 * h, p).view(hb.S, 3 * h)
            dm['seed'] = seeds[i]
            dm['dec_x'], dm['dec_xr'] = ms['dropout'][2 * i], ms['dropout'][2 * i + 1]
        out[rev] = dm
    return out


def place2(sub, uniq, N):
    """layer 2's compact-row mask on the whole graph's rows: node uniq[u] takes row u (rows no read-out reads stay 1)"""
    full = torch.ones(N, sub.shape[1], device=DEV)
    full[uniq] = sub
    return full


# ---- float64 restatement ------------------------------------------------------------------------------------------------------
def decode64(P, d, rev, r, mut=None, dm=None):
    """model.py:89-103 of one direction as restate.renet_forward restates them, the decoder inputs scaled by the recorded
    masks: loss_sub + 0.1 loss_sub_r"""
    R = d.R
    tr = d.trip
    if not rev:
        s, rr, o = tr[:, 0], tr[:, 1], tr[:, 2]
        rel = P['rel_embeds'][:R]
    else:
        o, rr, s = tr[:, 0], tr[:, 1], tr[:, 2]
        rel = P['rel_embeds'][:R] if mut == 'dec-rel-half' else P['rel_embeds'][R:]
    idx = np.arange(len(tr)) if mut == 'unsorted' else r.bh.s_idx
    s_t, r_t, o_t = enc._t(s[idx]), enc._t(rr[idx]), enc._t(o[idx])
    B = len(tr)
    pad = lambda x: torch.cat((x, x.new_zeros(B - len(x), x.shape[1])), 0)
    ent = P['ent_embeds'].detach() if mut == 'no-dec-ent-grad' else P['ent_embeds']
    x = torch.cat((ent[s_t], pad(r.s_h), rel[r_t]), 1)
    x_r = torch.cat((ent[s_t], pad(r.s_q)), 1)
    if dm is not None and 'dec_x' in dm:
        h2 = x_r.shape[1]
        x = x * dm['dec_x'].double()
        x_r = x_r * (dm['dec_x'][:, :h2] if mut == 'shared-mask' else dm['dec_xr']).double()
    loss = torch.nn.functional.cross_entropy(x @ P['linear.weight'].t() + P['linear.bias'], o_t)
    loss_r = torch.nn.functional.cross_entropy(x_r @ P['linear_r.weight'].t() + P['linear_r.bias'], r_t)
    return loss + (1.0 if mut == 'rel-weight' else 0.1) * loss_r


def encode64(P, d, rev, dm, mut=None):
    kw = {'mask1': dm['relu1']}
    if 'loop1' in dm:
        loop2 = place2(torch.roll(dm['sub2'], 1, 0), dm['uniq'], dm['N']) if mut == 'loop2-shift' else dm['loop2']
        x3 = dm['x4'].reshape(-1)[:dm['x3'].numel()].view_as(dm['x3']) if mut == 'x3-mask' else dm['x3']
        kw.update(loop1=dm['loop1'], loop2=loop2, x4=dm['x4'], x3=x3)
    return enc.restate_dir(P, d, rev, **kw)


def restate_step(P, d, masks, mut=None):
    """-> (loss_s, loss_o, {rev: restate_dir result})"""
    rs, losses = {}, []
    for rev in (False, True):
        rs[rev] = encode64(P, d, rev, masks[rev], mut)
        losses.append(decode64(P, d, rev, rs[rev], mut, masks[rev]))
    return losses[0], losses[1], rs


def params64(P):
    return {k: v.double().clone().requires_grad_(True) for k, v in P.items()}


def grads64(P, loss, keys, retain=True):
    g = torch.autograd.grad(loss, [P[k] for k in keys], retain_graph=retain, allow_unused=True)
    return {k: (x if x is not None else torch.zeros_like(P[k])) for k, x in zip(keys, g)}


def flat64(grads, lay, total):
    out = torch.zeros(total, dtype=torch.float64, device=DEV)
    for k, (o, n) in lay.items():
        out[o:o + n] = grads[k].reshape(-1)
    return out


# ---- bars -----------------------------------------------------------------------------------------------------------------------
def note(what, ratio, case):
    if ratio > WORST.get(what, (-1.0,))[0]:
        WORST[what] = (ratio, case)


def worst_rows(got, ref, tau):
    r = enc.row_ratio(got.reshape(len(got), -1) if got.dim() > 1 else got.reshape(1, -1),
                      ref.reshape(len(ref), -1) if ref.dim() > 1 else ref.reshape(1, -1), tau)
    return r


def check_rows(case, what, got, ref, tau):
    assert got.shape == ref.shape, (case, what, tuple(got.shape), tuple(ref.shape))
    assert torch.isfinite(got).all(), (case, what, 'not finite')
    r = worst_rows(got, ref, tau)
    worst = float(r.max()) if len(r) else 0.0
    note(what, worst, case)
    assert worst <= 1.0, '%s %s: row %d is %.3g x the bar off; %d of %d rows fail' % (
        case, what, int(r.argmax()), worst, int((r > 1).sum()), len(r))


def check_zero_rows(case, k, g, r):
    g, r = (g.reshape(1, -1), r.reshape(1, -1)) if r.dim() == 1 else (g, r)
    bad = (r == 0).all(1) & (g != 0).any(1)
    assert not bool(bad.any()), '%s d%s: row %d is exactly 0 in fp64 but not in the kernel\'s gradient' % (
        case, k, int(bad.nonzero()[0]))


def check_elems(case, what, got, ref, bound):
    err = (got.double() - ref).abs()
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, float('inf'), 0.0).double())
    worst = float(ratio.max())
    note(what, worst, case)
    i = int(ratio.argmax())
    assert worst <= 1.0, '%s %s: element %d is %.3g x its bound off (got %r, ref %r); %d elements fail' % (
        case, what, i, worst, float(got[i]), float(ref[i]), int((ratio > 1).sum()))


def loss_ratio(got, ref):
    return abs(float(got.detach()) - float(ref.detach())) / abs(float(ref.detach())) / LOSS_TOL


def grad_miss(gm, ref):
    return max(float(worst_rows(gm[k], ref[k], TAU_GRAD).max()) for k in ref)


def fwd_miss(rs_m, rs, revs=(False, True)):
    return max(max(float(enc.row_ratio(rs_m[v].s_h, rs[v].s_h, TAU_FWD).max()),
                   float(enc.row_ratio(rs_m[v].s_q, rs[v].s_q, TAU_FWD).max())) for v in revs)


def adam_miss(mut, ref_pmv, bounds):
    return max(float(((a - b).abs() / bd.clamp_min(1e-300)).max()) for a, b, bd in zip(mut, ref_pmv, bounds))


# ---- one step against fp64 ----------------------------------------------------------------------------------------------------------
def check_step(case, k, st, prev, p, max_norm, regime, required, lay, total):
    """restate step k, show the mistakes (when required is not None), then compare everything the step computed"""
    tag = '%s-step%d' % (case, k)
    d = st.d
    masks = masks_of(tag, st, p)
    for rev in (False, True):
        hb, dm = masks[rev]['hb'], masks[rev]
        lens = d.lens(rev)
        np.testing.assert_array_equal(np.asarray(hb.s_idx), np.argsort(-lens, kind='stable'), err_msg=tag + ' s_idx')
    P = params64(st.P)
    keys = list(lay)
    loss_s, loss_o, rs = restate_step(P, d, masks)
    for rev in (False, True):
        assert np.array_equal(masks[rev]['hb'].graph.node_ent.cpu().numpy(), rs[rev].g.id), 'the batchers number nodes differently'
    loss64 = loss_s + loss_o
    g_s = grads64(P, loss_s, keys)
    g_o = grads64(P, loss_o, keys)
    ref = {k2: g_s[k2] + g_o[k2] for k2 in keys}
    g64 = flat64(ref, lay, total)
    # ---- the clip regime and the Adam restatement of the kernel's gradient
    o = st.opt
    G = o['g']
    ssq = float((G.double() ** 2).sum())
    coef = sup.f32(max_norm) / (np.sqrt(ssq) + 1e-6)
    if regime == 'clip':
        assert coef < 1.0 / REGIME_MARGIN, (tag, 'expected to clip', coef)
    else:
        assert coef > REGIME_MARGIN, (tag, 'expected no clipping', coef)
    clip = sup.clip_coef(o['sumsq'], max_norm)
    adam = lambda g, step=o['step'], wd=WD, c=clip: sup.adam_ref(o['p'], g, o['m'], o['v'], step, c, LR, BETAS[0], BETAS[1],
                                                                 EPS, wd)
    pmv, bounds = adam(G)
    # ---- mistakes
    if required is not None:
        got = {}
        with torch.no_grad():
            for mut in ('x3-mask', 'loop2-shift'):
                if p:
                    rev = mut == 'loop2-shift'
                    rm = encode64(P, d, rev, masks[rev], mut)
                    got[mut] = fwd_miss({rev: rm}, rs, (rev,))
            if prev is not None:
                Pp = params64(prev.P)
                ls, lo, rsm = restate_step(Pp, d, masks)
                got['stale'] = max(loss_ratio(ls + lo, loss64), fwd_miss(rsm, rs))
        for mut in DEC_MUTS:
            if mut == 'shared-mask' and not p:
                continue
            lm = [decode64(P, d, rev, rs[rev], mut, masks[rev]) for rev in (False, True)]
            tot = lm[0] if mut == 'drop-obj-loss' else lm[0] + lm[1]
            got[mut] = max(loss_ratio(tot, loss64), grad_miss(grads64(P, tot, keys), ref))
        ref64 = adam(g64, c=sup.clip_coef(float((g64 ** 2).sum()), max_norm))[0]
        got['adam-no-wd'] = adam_miss(adam(g64, wd=0.0, c=sup.clip_coef(float((g64 ** 2).sum()), max_norm))[0], ref64, bounds)
        got['adam-bias-step'] = adam_miss(adam(g64, step=o['step'] + 1, c=sup.clip_coef(float((g64 ** 2).sum()), max_norm))[0],
                                          ref64, bounds)
        fs, fo = flat64(g_s, lay, total), flat64(g_o, lay, total)
        per_dir = sup.clip_coef(float((fs ** 2).sum()), max_norm) * fs + sup.clip_coef(float((fo ** 2).sum()), max_norm) * fo
        if regime == 'clip':
            got['clip-per-dir'] = adam_miss(adam(per_dir, c=1.0)[0], ref64, bounds)
        for kind in required:
            assert kind in got, '%s: the case cannot express the mistake %s' % (tag, kind)
            assert got[kind] >= MISS, '%s: the mistake %s misses the bar by only %.3g x' % (tag, kind, got[kind])
            if got[kind] < MISSES.get(kind, (float('inf'),))[0]:
                MISSES[kind] = (got[kind], tag)
    # ---- loss, encoder rows, gradient rows
    lerr = loss_ratio(st.loss, loss64)
    note('loss (rel err / 1e-5)', lerr, tag)
    assert lerr <= 1.0, (tag, 'loss', float(st.loss), float(loss64.detach()))
    for rev in (False, True):
        dm, r = masks[rev], rs[rev]
        check_rows(tag + ('-obj' if rev else '-subj'), 's_h', dm['s_h'], r.s_h.detach(), TAU_FWD)
        check_rows(tag + ('-obj' if rev else '-subj'), 's_q', dm['s_q'], r.s_q.detach(), TAU_FWD)
    named = dict(st.P)
    assert set(named) == set(lay), (tag, 'parameters outside the flat buffers', set(named) ^ set(lay))
    for k2, (off, n) in lay.items():
        g = G[off:off + n].view(named[k2].shape)
        check_zero_rows(tag, k2, g, ref[k2])
        check_rows(tag, 'd' + k2, g, ref[k2], TAU_GRAD)
    # ---- the flat buffers and the step
    assert o['sumsq'] >= 0
    L = sup.sumsq_terms(total)[1]
    sup_bar = (L + 24) * sup.U * ssq
    note('grad sumsq (err / bar)', abs(o['sumsq'] - ssq) / sup_bar, tag)
    assert abs(o['sumsq'] - ssq) <= sup_bar, (tag, 'sum of squares', o['sumsq'], ssq)
    for what, got_, r_, b_ in zip(('adam p', 'adam m', 'adam v'), (st.after['flat_p'], st.after['exp_avg'], st.after['exp_avg_sq']),
                                  pmv, bounds):
        check_elems(tag, what, got_, r_, b_)
    pad = torch.ones(total, dtype=torch.bool, device=DEV)
    for off, n in lay.values():
        pad[off:off + n] = False
    for what, buf in (('flat_p', st.after['flat_p']), ('exp_avg', st.after['exp_avg']), ('exp_avg_sq', st.after['exp_avg_sq']),
                      ('flat_g', G)):
        assert bool((buf[pad] == 0).all()), (tag, 'ALIGN padding of %s is not 0' % what)


def check_aliasing(case, m, tr, lay, total):
    assert tr.total == total and tr.flat_p.numel() == total, (case, 'flat buffer size', tr.total, total)
    base_p, base_g = tr.flat_p.data_ptr(), tr.flat_g.data_ptr()
    for k, p in m.named_parameters():
        off, n = lay[k]
        assert p.data_ptr() == base_p + 4 * off and p.is_contiguous(), (case, k, 'does not alias flat_p at its offset')
        assert p.grad is not None and p.grad.data_ptr() == base_g + 4 * off, (case, k, '.grad does not alias flat_g')


# ---- which kernels ran ------------------------------------------------------------------------------------------------------------
def gather_choice(E, N, indexed):
    """rgcn_fwd.cu's gather_use_stream for h = 200 (common.cuh's thresholds)"""
    min_nodes = 16384 if indexed else 2048
    return 'stream' if E >= 16384 and min_nodes <= N <= 40960 else 'tile'


def forward_gathers(names):
    return {x for x in glb.rgcn_kernels(names)
            if x[0] == 'rgcn_gather_d200_kernel' or (x[0] == 'rgcn_gather_stream_kernel' and not x[1][3])}


def assert_served(case, fn, layers, p, det):
    """layers: the forward gathers ('stream' / 'tile') for layers 1 and 2"""
    exp = {x for x in glb.expected_rgcn(*layers)}
    want = ['ce_reduce_kernel']
    if p:
        want += ['pack_inputs_dropout_kernel'] + (['dropout_grad_rows_kernel', 'scatter_add_rows_sorted_kernel'] if det else
                                                  ['unpack_inputs_dropout_kernel'])
    ce = [r'umma_gemm_packed_kernel<(false|\(bool\)0), (\(int\))?1>', r'umma_gemm_packed_kernel<(false|\(bool\)0), (\(int\))?2>']

    def done(names):
        sn = glb.short_names(names)
        return all(w in sn for w in want) and all(any(re.search(c, n) for n in names) for c in ce) and exp <= forward_gathers(names)
    names = glb.trace(fn, want=done)
    sn = glb.short_names(names)
    for w in want:
        assert w in sn, '%s: %s did not run (%s)' % (case, w, sorted(sn))
    for c in ce:
        assert any(re.search(c, n) for n in names), '%s: no kernel matches %s' % (case, c)
    if not p:
        assert 'pack_inputs_dropout_kernel' not in sn, (case, 'the dropout GRU path ran at p = 0')
    if det:
        assert 'unpack_inputs_dropout_kernel' not in sn, (case, 'the atomic dropout scatter ran in deterministic mode')
    rnn = sorted(n for n in names if re.search(r'cudnn|[Rr][Nn][Nn]', n))
    assert not rnn, (case, 'a cuDNN RNN kernel ran', rnn[:3])
    seen = forward_gathers(names)
    assert seen == exp, '%s: forward gathers %s, expected %s' % (case, sorted(seen), sorted(exp))


# ---- a case ---------------------------------------------------------------------------------------------------------------------
def run_case(case, batches, layers, p=P_DROP, feed='views', det=False, max_norm=CLIP_NORM, regime='clip', required=None, seed=0):
    """layers: the forward gathers ('stream' / 'tile') of layers 1 and 2 on the last batch"""
    from rgcn_contract_check import deterministic
    t0 = time.perf_counter()
    if required is None:
        required = ALL_MUTS if p else NO_DROPOUT_MUTS
    required = tuple(k for k in required if k != 'stale' or len(batches) > 1)
    required = tuple(k for k in required if k != 'clip-per-dir' or regime == 'clip')
    mode = (lambda: deterministic(True)) if det else contextlib.nullcontext

    def steps():
        m = make_model(batches[0], p, seed)
        m.train()
        tr, cap = make_trainer(m, max_norm)
        lay, total = layout(m)
        check_aliasing(case, m, tr, lay, total)
        with mode():
            out = run_steps(m, tr, batches, feed, cap)
        check_aliasing(case, m, tr, lay, total)
        return m, tr, out, lay, total
    m, tr, out, lay, total = steps()
    if det:
        _, tr2, again, _, _ = steps()
        for k, (a, b) in enumerate(zip(out, again)):
            assert torch.equal(a.loss, b.loss), (case, k, 'deterministic mode: the loss differs between runs')
            assert torch.equal(a.opt['g'], b.opt['g']), (case, k, 'deterministic mode: flat_g differs between runs')
            assert torch.equal(a.after['flat_p'], b.after['flat_p']), (case, k, 'deterministic mode: flat_p differs')
        tr2.close()
    # ---- which gather each layer runs on the last batch (the one traced below): the dispatch rule for the recorded sizes
    # must give what the case states
    for rev in (False, True):
        _, N1, E1 = out[-1].rec['l1'][int(rev)]
        _, N2, E2 = out[-1].rec['l2'][int(rev)]
        rule = (gather_choice(E1, N1, True), gather_choice(E2, N2, False))
        assert rule == tuple(layers), (case, 'the dispatch rule gives', rule, 'for (N1, E1, S, E2)', (N1, E1, N2, E2))
    disc = 1 if len(out) > 1 else 0
    for k, st in enumerate(out):
        check_step(case, k, st, out[k - 1] if k else None, p, max_norm, regime, required if k == disc else None, lay, total)
    # ---- which kernels ran: a further step on the last batch
    from renet_b200.parallel import native_optimizer_step
    tr.optimizer_step = native_optimizer_step
    d = batches[-1]
    sh, oh, gd = (out[-1].rec['enc'][0][2], out[-1].rec['enc'][1][2], None) if feed == 'prefetch' else inputs_of(d, feed)
    q = torch.from_numpy(d.trip).to(DEV)
    with mode():
        assert_served(case, lambda: tr.train_step(q, sh, oh, gd), layers, p, det)
    tr.close()
    SECONDS[case] = time.perf_counter() - t0


# ---- the cases ------------------------------------------------------------------------------------------------------------------
CASES = {}


def case(name):
    def reg(fn):
        assert name not in CASES

        def run():
            fn(name)
        CASES[name] = run
        return fn
    return reg


def batches_of(preset, seed, T, B, idx=(0, 1, 2)):
    t = enc.tkg(preset, seed, T)
    return [enc.tkg_data(preset, seed, T, t.batch_indices(i, B)) for i in idx]


def bench_batches():
    return batches_of('icews18', 999, 240, 1024)


@case('icews18-bench')
def _(cs):
    """the benchmark's batches (ICEWS18 shape, 240 timestamps, batch 1024) at dropout 0.5 through the device batcher"""
    run_case(cs, bench_batches(), layers=('stream', 'stream'))


@case('icews18-bench-p0')
def _(cs):
    """the same batches at dropout 0: the split GI / PQ / PT GRU path, the configuration bench.py times (max_norm 1, which
    these steps' gradients stay below)"""
    run_case(cs, bench_batches(), ('stream', 'stream'), p=0.0, max_norm=1.0, regime='none')


@case('icews18-prefetched')
def _(cs):
    """HistoryBatches from hoststore.prefetch, fed to train_step as bench.py's train_region feeds its batches"""
    run_case(cs, bench_batches(), feed='prefetch', layers=('stream', 'stream'), seed=1)


@case('gdelt')
def _(cs):
    """GDELT shape, batch 1024: many small components, layer 1 under the stream kernel's node threshold"""
    run_case(cs, batches_of('gdelt', 5, 60, 1024), ('tile', 'stream'), seed=2)


@case('icews14')
def _(cs):
    """ICEWS14 shape, batch 1024: about 12 k layer-1 nodes, so layer 1 on the tile kernel and layer 2 on the stream kernel"""
    run_case(cs, batches_of('icews14', 3, 60, 1024), ('tile', 'stream'), seed=3)


def ragged_data(B, seed):
    """B samples of the ICEWS18-shaped stream: some with an empty history in one direction only, a subject twice, one
    triple twice, and a last sample (s, R - 1, N - 1) with s's history and no object history"""
    t = enc.tkg('icews18', 7, 40)
    rng = np.random.default_rng(seed)
    ls = np.asarray([len(x) for x in t.s_hist])
    lo = np.asarray([len(x) for x in t.o_hist])
    only_s = rng.choice(np.flatnonzero((ls > 0) & (lo == 0)), 3, replace=False)
    only_o = rng.choice(np.flatnonzero((ls == 0) & (lo > 0)), 3, replace=False)
    both = np.flatnonzero((ls > 0) & (lo > 0))
    subj = t.quads[both, 0]
    vals, cnt = np.unique(subj, return_counts=True)
    twice = both[subj == vals[np.argmax(cnt)]][:2]
    rest = rng.choice(np.setdiff1d(both, np.concatenate((only_s, only_o, twice))), B - 10, replace=False)
    sel = np.concatenate((only_s[:1], rest[:B // 3], only_o, twice, rest[B // 3:], only_s[1:], rest[:1]))
    last = int(twice[0])
    trip = np.concatenate((t.quads[sel, :3], [[t.quads[last, 0], t.num_r - 1, t.num_e - 1]]))
    hists = {False: ([t.s_hist[i] for i in sel] + [t.s_hist[last]], [t.s_hist_t[i] for i in sel] + [t.s_hist_t[last]]),
             True: ([t.o_hist[i] for i in sel] + [[]], [t.o_hist_t[i] for i in sel] + [[]])}
    d = enc.Data(t.quads, t.num_e, t.num_r, 200, 100, np.arange(len(trip)), hists, t.global_emb, trip=trip)
    assert len(d.trip) == B, (len(d.trip), B)
    return d


@case('ragged')
def _(cs):
    """B = 37, 1000 and 37 (other samples)"""
    batches = [ragged_data(37, 1), ragged_data(1000, 2), ragged_data(37, 3)]
    for d in batches:
        ls, lo = d.lens(False), d.lens(True)
        assert ((ls > 0) & (lo == 0)).any() and ((ls == 0) & (lo > 0)).any(), 'no one-sided empty history'
        full = d.trip[(ls > 0)]
        assert len(np.unique(full[:, 0])) < len(full), 'no duplicate subject'
        assert len(np.unique(d.trip, axis=0)) < len(d.trip), 'no duplicated triple'
        assert d.trip[:, 2].max() == d.num_e - 1 and d.trip[:, 1].max() == d.R - 1, 'labels N - 1 / R - 1 missing'
    run_case(cs, batches, layers=('tile', 'tile'), seed=4)


@case('clip-inactive')
def _(cs):
    """the benchmark's batches with max_norm far above the gradient norm"""
    run_case(cs, bench_batches(), max_norm=1e3, regime='none', layers=('stream', 'stream'), seed=5)


@case('det')
def _(cs):
    """dropout 0.5 under torch.use_deterministic_algorithms(True): two runs from the same seeds bitwise equal"""
    run_case(cs, bench_batches(), det=True, layers=('stream', 'stream'), seed=6)


@case('lists')
def _(cs):
    """the reference's list inputs: the numpy batcher, one step"""
    run_case(cs, bench_batches()[:1], feed='lists', layers=('stream', 'stream'), seed=7)


def summary():
    out = ['%-34s worst err/bar %.3f  (%s)' % (w, v[0], v[1]) for w, v in sorted(WORST.items())]
    out += ['mistake %-16s smallest miss %.3g x the bar  (%s)' % (k, v[0], v[1]) for k, v in sorted(MISSES.items())]
    out += ['%-28s %.1f s' % (k, v) for k, v in sorted(SECONDS.items())]
    return out
