"""Run in a subprocess by tests/test_gpu_gru_contract.py: the fused read-out + GRU forward and backward (renet_gru_fwd /
renet_gru_bwd, and the dropout and dense entries) against a float64 autograd reference at the recurrence's schedule edges.

The sequence structure is built here directly, not by the batcher, so that the sequence count Q, the lengths and the
per-step active counts (host_batch_sizes) can be chosen freely.  The persistent recurrence kernel runs a grid of
(7 unit slices, 2 encoders, gz) CTAs with gz = min(m-tiles, 132 / 14) = 9 at h = 200, so a CTA walks a second 128-row
m-tile only when Q > 9 * 128 = 1152: Q = 1153 and 3000 reach the second and third.  Ragged lengths make the active count
drop across multiples of 128 between steps; length 16 is the longest sequence the workspaces hold.  h = 400 (the kernel
takes h <= 224), h = 100 (3h % 200 != 0: weights packed for sgemm_nn) and engine 0 run the step-by-step loop instead.

Forward: hn4 / hn3 start as NaN; every row must be written and match within 1e-4 (max-abs-diff / max-abs-ref).
Backward: dH2 is written (starts as NaN) and must match within 2e-4.  Every accumulated gradient -- d_ent, d_rel, d_glob
and the eight GRU parameter gradients -- starts from a random non-zero base and must equal base + reference within 2e-4
of the reference gradient's largest element."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import restate  # noqa: E402
from renet_b200 import _lib  # noqa: E402

L, P = _lib.lib(), _lib.ptr
dev = 'cuda:0'
F64 = torch.float64
# forward launches before the recurrence on the tensor-core path (packed-weight cache off): 9 weight packs, 2 bias rows,
# the GI / PQ (entity, relation) / PT projections
PRELUDE = 15

stream = _lib.stream()
L.renet_set_weight_generation(-1)
worst = {'fwd': 0.0, 'bwd': 0.0}
n_cases = 0


def err(got, ref):
    return ((got.double() - ref).abs().max() / ref.abs().max()).item()


def lens_from_batch_sizes(bs):
    """Per-sequence lengths (sorted descending) whose active count at step t is bs[t]."""
    bs = np.asarray(bs)
    return np.array([int((bs > q).sum()) for q in range(int(bs[0]))], dtype=np.int64)


def case(name, h, lens, T, engine=1, recur=None, p_drop=0.0, dense=False):
    global n_cases
    torch.manual_seed(n_cases)
    n_cases += 1
    lens = np.asarray(lens, dtype=np.int64)
    assert np.all(np.diff(lens) <= 0) and lens.min() >= 1
    Q, S, max_len = len(lens), int(lens.sum()), int(lens.max())
    bs = np.array([int((lens > t).sum()) for t in range(max_len)], dtype=np.int32)
    starts = np.concatenate(([0], np.cumsum(lens)[:-1])).astype(np.int32)
    num_e, num_r, NH = 5000, 460, max(S // 2, 1)
    g = lambda *s, sc=1.0: (torch.randn(*s, device=dev) * sc)
    i32 = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.int32, device=dev)
    H2, ent, rel, glob = g(NH, h, sc=0.5), g(num_e, h, sc=0.3), g(num_r, h, sc=0.3), g(T, h, sc=0.1)
    readout = torch.randint(0, NH, (S,), device=dev, dtype=torch.int32)        # read-out rows with repeats
    row_glob = torch.randint(0, T, (S,), device=dev, dtype=torch.int32)
    seq_s = torch.randint(0, num_e, (Q,), device=dev, dtype=torch.int32)
    seq_r = torch.randint(0, num_r, (Q,), device=dev, dtype=torch.int32)
    row_seq = i32(np.repeat(np.arange(Q), lens))
    seq_len, seq_start = i32(lens), i32(starts)
    k4 = h if dense else 4 * h
    sc = 1.0 / h ** 0.5
    w_ih4, w_hh4, b_ih4, b_hh4 = g(3 * h, k4, sc=sc), g(3 * h, h, sc=sc), g(3 * h, sc=0.1), g(3 * h, sc=0.1)
    w_ih3, w_hh3, b_ih3, b_hh3 = g(3 * h, 3 * h, sc=sc), g(3 * h, h, sc=sc), g(3 * h, sc=0.1), g(3 * h, sc=0.1)
    X4d = g(S, k4, sc=0.5) if dense else None

    # ---- fp64 reference with autograd
    leaves = [t.double().requires_grad_(True) for t in (H2, ent, rel, glob, w_ih4, w_hh4, b_ih4, b_hh4, w_ih3, w_hh3, b_ih3,
                                                         b_hh3)]
    H2r, entr, relr, globr, wi4, wh4, bi4, bh4, wi3, wh3, bi3, bh3 = leaves
    mask4 = mask3 = None
    if p_drop > 0:
        seed = 987654321 + n_cases
        m = torch.empty(S * 7 * h, device=dev)
        _lib.check(L.renet_dropout_mask(seed, 0, m.numel(), p_drop, P(m), stream), 'renet_dropout_mask')
        mask4, mask3 = m[:S * 4 * h].view(S, 4 * h).double(), m[S * 4 * h:].view(S, 3 * h).double()
    if dense:
        X4r = X4d.double().requires_grad_(True)
        ref4 = restate.gru_final_hidden_batched(X4r, lens, wi4, wh4, bi4, bh4)
        ref3 = None
    else:
        X4, X3, _, _ = restate.packed_inputs(H2r, readout.long(), lens, seq_s.long(), seq_r.long(), entr, relr,
                                             globr[row_glob.long()])
        if mask4 is not None:
            X4, X3 = X4 * mask4, X3 * mask3
        ref4 = restate.gru_final_hidden_batched(X4, lens, wi4, wh4, bi4, bh4)
        ref3 = restate.gru_final_hidden_batched(X3, lens, wi3, wh3, bi3, bh3)
    dhn4, dhn3 = g(Q, h), (torch.zeros(Q, h, device=dev) if dense else g(Q, h))
    loss = (ref4 * dhn4.double()).sum() + (0 if dense else (ref3 * dhn3.double()).sum())
    loss.backward()

    # ---- forward through the C-ABI
    L.renet_set_gemm_engine(engine)
    try:
        hn4 = torch.full((Q, h), float('nan'), device=dev)
        hn3 = torch.full((Q, h), float('nan'), device=dev)
        hbs = bs.ctypes.data_as(_lib.ctypes.c_void_p)
        weights = [P(t) for t in (w_ih4, w_hh4, b_ih4, b_hh4, w_ih3, w_hh3, b_ih3, b_hh3)]
        if dense:
            nbytes = int(L.renet_gru_dropout_workspace_bytes(S, Q, 1, h))
        elif p_drop > 0:
            nbytes = int(L.renet_gru_dropout_workspace_bytes(S, Q, T, h))
        else:
            nbytes = int(L.renet_gru_workspace_bytes(S, Q, T, h))
        ws = torch.empty(nbytes // 4, device=dev)
        n0 = _lib.launch_count()
        if dense:
            rc = L.renet_gru_dense_fwd(P(X4d), k4, None, 0, P(seq_len), P(seq_start), hbs, max_len, *weights[:4], None, None, None,
                                       None, P(hn4), P(hn3), S, Q, h, P(ws), nbytes, stream)
        elif p_drop > 0:
            rc = L.renet_gru_fwd_dropout(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel), P(row_seq), P(seq_s), P(seq_r),
                                         P(seq_len), P(seq_start), hbs, max_len, *weights, P(hn4), P(hn3), S, Q, T, h, p_drop,
                                         seed, P(ws), nbytes, stream)
        else:
            rc = L.renet_gru_fwd(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel), P(seq_s), P(seq_r), P(seq_len),
                                 P(seq_start), hbs, max_len, *weights, P(hn4), P(hn3), S, Q, T, h, P(ws), nbytes, stream)
        _lib.check(rc, 'gru forward (%s)' % name)
        launches = _lib.launch_count() - n0
        torch.cuda.synchronize()
        if recur is not None:
            # one cooperative launch for every step, or per step one gate kernel plus (t > 0) the recurrent product(s)
            if recur:
                assert launches == PRELUDE + 1, '%s: %d forward launches, not the recurrence kernel' % (name, launches)
            else:
                assert launches >= PRELUDE + 2 * max_len - 1, '%s: %d forward launches, not the step loop' % (name, launches)
        assert not torch.isnan(hn4).any() and (dense or not torch.isnan(hn3).any()), '%s: hidden states left unwritten' % name
        e_f = max(err(hn4, ref4.detach()), 0.0 if dense else err(hn3, ref3.detach()))
        assert e_f < 1e-4, '%s: forward error %.3e' % (name, e_f)

        # ---- backward: written outputs start as NaN, accumulated ones from a random base
        base = lambda t: torch.randn_like(t)
        grads_ref = {'w_ih4': wi4.grad, 'w_hh4': wh4.grad, 'b_ih4': bi4.grad, 'b_hh4': bh4.grad}
        if not dense:
            grads_ref.update({'d_ent': entr.grad, 'd_rel': relr.grad, 'd_glob': globr.grad, 'w_ih3': wi3.grad, 'w_hh3': wh3.grad,
                              'b_ih3': bi3.grad, 'b_hh3': bh3.grad})
        acc = {k: base(v.float()) for k, v in grads_ref.items()}
        start = {k: v.clone() for k, v in acc.items()}
        wb = [P(t) for t in (w_ih4, w_hh4, w_ih3, w_hh3)]
        dw = [P(acc.get(k)) for k in ('w_ih4', 'w_hh4', 'b_ih4', 'b_hh4', 'w_ih3', 'w_hh3', 'b_ih3', 'b_hh3')]
        if dense:
            bbytes = int(L.renet_gru_bwd_dropout_workspace_bytes(S, Q, 1, h))
            bws = torch.empty(bbytes // 4, device=dev)
            dX4 = torch.full((S, k4), float('nan'), device=dev)
            rc = L.renet_gru_dense_bwd(P(X4d), k4, None, 0, P(seq_len), P(seq_start), hbs, max_len, wb[0], wb[1], None, None,
                                       P(dhn4), P(dhn3), P(dX4), None, *dw[:4], None, None, None, None, S, Q, h, P(ws), P(bws),
                                       bbytes, stream)
            written = {'dX4': (dX4, X4r.grad)}
        else:
            dH2 = torch.full((NH, h), float('nan'), device=dev)
            if p_drop > 0:
                bbytes = int(L.renet_gru_bwd_dropout_workspace_bytes(S, Q, T, h))
                bws = torch.empty(bbytes // 4, device=dev)
                rc = L.renet_gru_bwd_dropout(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel), P(row_seq), P(seq_s),
                                             P(seq_r), P(seq_len), P(seq_start), hbs, max_len, *wb, P(dhn4), P(dhn3), P(dH2),
                                             P(acc['d_ent']), P(acc['d_rel']), P(acc['d_glob']), *dw, NH, S, Q, T, h, p_drop,
                                             seed, P(ws), P(bws), bbytes, stream)
            else:
                bbytes = int(L.renet_gru_bwd_workspace_bytes(S, Q, T, h))
                bws = torch.empty(bbytes // 4, device=dev)
                rc = L.renet_gru_bwd(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel), P(seq_s), P(seq_r), P(seq_len),
                                     P(seq_start), hbs, max_len, *wb, P(dhn4), P(dhn3), P(dH2), P(acc['d_ent']),
                                     P(acc['d_rel']), P(acc['d_glob']), *dw, NH, S, Q, T, h, P(ws), P(bws), bbytes, stream)
            written = {'dH2': (dH2, H2r.grad)}
        _lib.check(rc, 'gru backward (%s)' % name)
        torch.cuda.synchronize()
    finally:
        L.renet_set_gemm_engine(1)
    e_b, which = 0.0, ''
    for k, (got, ref) in written.items():
        assert not torch.isnan(got).any(), '%s: %s left unwritten' % (name, k)
        e = err(got, ref)
        if e > e_b:
            e_b, which = e, k
    for k, ref in grads_ref.items():
        # the accumulated result against base + reference, relative to the reference gradient itself
        e = ((acc[k].double() - start[k].double() - ref).abs().max() / ref.abs().max()).item()
        if e > e_b:
            e_b, which = e, k
    assert e_b < 2e-4, '%s: backward error %.3e in %s' % (name, e_b, which)
    worst['fwd'], worst['bwd'] = max(worst['fwd'], e_f), max(worst['bwd'], e_b)
    path = '' if recur is None else ('recurrence kernel' if recur else 'step loop')
    print('%-40s h=%-3d Q=%-5d S=%-6d T=%-3d L=%-2d %-18s fwd %.2e bwd %.2e (%s)' % (
        name, h, Q, S, T, max_len, path, e_f, e_b, which), flush=True)


RAGGED_3000 = [3000, 1153, 1153, 640, 640, 129, 128, 127, 64, 64, 1, 1, 1, 1, 1, 1]   # n_act across multiples of 128
ones, sixteen = (lambda Q: [1] * Q), (lambda Q: [16] * Q)

# ---- h = 200, the persistent recurrence kernel
case('one sequence, length 16', 200, sixteen(1), 1, recur=True)
case('one sequence, length 1', 200, ones(1), 37, recur=True)
case('Q = 127 ragged', 200, lens_from_batch_sizes([127, 127, 100, 64, 63, 1]), 37, recur=True)
case('Q = 128 lengths 1', 200, ones(128), 37, recur=True)
case('Q = 129 lengths 16', 200, sixteen(129), 1, recur=True)
case('Q = 1152 ragged', 200, lens_from_batch_sizes([1152, 1152, 640, 129, 128, 127, 64, 1]), 37, recur=True)
case('Q = 1153 lengths 16 (second m-tile)', 200, sixteen(1153), 37, recur=True)
case('Q = 1153 lengths 1', 200, ones(1153), 1, recur=True)
case('Q = 3000 ragged (third m-tile)', 200, lens_from_batch_sizes(RAGGED_3000), 37, recur=True)
case('Q = 3000 lengths 16', 200, sixteen(3000), 37, recur=True)
# ---- the step-by-step loop
case('engine 0 (FFMA projections + loop)', 200, lens_from_batch_sizes([1153, 640, 129, 128, 127, 64, 1]), 37, engine=0,
     recur=False)
case('h = 400 (batched streaming GEMM loop)', 400, lens_from_batch_sizes([1153, 640, 129, 128, 127, 64, 1]), 37, recur=False)
case('h = 100 (sgemm_nn weights, loop)', 100, lens_from_batch_sizes([300, 300, 129, 128, 1]), 13, recur=False)
# ---- input dropout (masks from renet_dropout_mask) and the dense single GRU
case('dropout p = 0.5, Q = 1153', 200, lens_from_batch_sizes([1153, 1153, 640, 129, 1]), 37, p_drop=0.5)
case('dense k4 = h, X3 = NULL', 200, lens_from_batch_sizes([1153, 640, 129, 128, 1]), 1, dense=True)

# ---- max_len = 17: rejected before anything is launched or written
h, Q, S, T = 200, 4, 68, 1
bs = np.array([4] * 17, dtype=np.int32)
z = lambda *s: torch.zeros(*s, device=dev)
zi = lambda n: torch.zeros(n, dtype=torch.int32, device=dev)
W = [z(3 * h, 4 * h), z(3 * h, h), z(3 * h), z(3 * h), z(3 * h, 3 * h), z(3 * h, h), z(3 * h), z(3 * h)]
hn = torch.full((Q, h), float('nan'), device=dev)
nb = int(L.renet_gru_workspace_bytes(S, Q, T, h))
ws = torch.empty(nb // 4, device=dev)
n0 = _lib.launch_count()
rc = L.renet_gru_fwd(P(z(S, h)), P(zi(S)), P(zi(S)), P(z(T, h)), P(z(1, h)), P(z(1, h)), P(zi(Q)), P(zi(Q)), P(zi(Q) + 17),
                     P(zi(Q)), bs.ctypes.data_as(_lib.ctypes.c_void_p), 17, *[P(t) for t in W], P(hn), P(hn), S, Q, T, h, P(ws), nb,
                     stream)
assert rc == -1 and b'max_len' in L.renet_last_error(), (rc, L.renet_last_error())
bb = int(L.renet_gru_bwd_workspace_bytes(S, Q, T, h))
dH2 = torch.full((S, h), float('nan'), device=dev)
rc = L.renet_gru_bwd(P(z(S, h)), P(zi(S)), P(zi(S)), P(z(T, h)), P(z(1, h)), P(z(1, h)), P(zi(Q)), P(zi(Q)), P(zi(Q) + 17),
                     P(zi(Q)), bs.ctypes.data_as(_lib.ctypes.c_void_p), 17, P(W[0]), P(W[1]), P(W[4]), P(W[5]), P(z(Q, h)),
                     P(z(Q, h)), P(dH2), P(z(1, h)), P(z(1, h)), P(z(T, h)), *[P(z(*t.shape)) for t in W], S, S, Q, T, h, P(ws),
                     P(torch.empty(bb // 4, device=dev)), bb, stream)
assert rc == -1 and b'max_len' in L.renet_last_error(), (rc, L.renet_last_error())
torch.cuda.synchronize()
assert _lib.launch_count() == n0 and torch.isnan(hn).all() and torch.isnan(dH2).all(), 'max_len 17 launched or wrote'
print('max_len = 17 rejected by forward and backward, nothing launched or written')
print('GRU_CONTRACT_OK %d cases, worst fwd %.2e bwd %.2e' % (n_cases, worst['fwd'], worst['bwd']))
