"""The global model's pre-training epoch on the kernels: the soft-target cross-entropy on the wgmma decoder
(renet_decoder_soft_ce_fwd/_bwd, decoder.decoder_soft_cross_entropy) against fp64 PyTorch, the batched
RENet_global.get_global_emb against the per-timestamp predict loop it replaces, and the pre-training step (pretrain.py:83-86)
through DataParallelTrainer without cuBLAS, bitwise reproducible, and data parallel."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_deterministic_sass import FLOAT_ATOMIC, sass  # noqa: F401  (sass is a fixture)

DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


def _soft_targets(M, N, gen):
    """Sparse normalised rows, each with mass in the last class tile; row 1 all zero, the last row sums to 1.7."""
    P = torch.zeros(M, N)
    last_tile = (N - 1) // 200 * 200
    for i in range(M):
        cols = torch.cat((torch.randint(0, N, (6,), generator=gen), torch.randint(last_tile, N, (2,), generator=gen)))
        P[i, cols] += torch.rand(8, generator=gen) + 0.05
        P[i] /= P[i].sum()
    if M > 2:
        P[1] = 0
    if M > 1:
        P[-1] *= 1.7
    return P


def _reference(x, w, b, P):
    logp = torch.nn.functional.log_softmax(torch.nn.functional.linear(x, w, b), dim=1)
    return torch.mean(torch.sum(-P * logp, 1))


@gpu
@pytest.mark.parametrize('M,N,K', [(1024, 23033, 200), (1024, 7691, 200), (240, 23033, 200), (37, 1001, 24), (1, 199, 8)])
def test_fused_soft_cross_entropy_vs_torch_fp64(M, N, K):
    from renet_b200.decoder import decoder_soft_cross_entropy
    gen = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=gen) * 0.5
    w = torch.randn(N, K, generator=gen) * (1.0 / K ** 0.5)
    b = torch.randn(N, generator=gen) * 0.1
    P = _soft_targets(M, N, gen).double()                  # the reference's targets are fp64
    xr, wr, br = (t.double().to(DEV).requires_grad_(True) for t in (x, w, b))
    ref = _reference(xr, wr, br, P.to(DEV))
    (0.7 * ref).backward()
    ref = float(ref.detach())
    runs = []
    for _ in range(2):
        xs, ws_, bs = (t.to(DEV).requires_grad_(True) for t in (x, w, b))
        loss = decoder_soft_cross_entropy(xs, ws_, bs, P.to(DEV))
        assert loss.dtype == torch.float64 and loss.dim() == 0
        (0.7 * loss).backward()
        runs.append([loss.detach(), xs.grad, ws_.grad, bs.grad])
    assert abs(float(runs[0][0]) - ref) < 1e-5 * abs(ref), (float(runs[0][0]), ref)
    for a, r, nm in zip(runs[0][1:], (xr.grad, wr.grad, br.grad), ('dX', 'dW', 'db')):
        err = float((a.double() - r).abs().max() / r.abs().max())
        assert err < 1e-4, (nm, err)
    for a, c in zip(*runs):
        assert torch.equal(a, c)


# ---- the embedding table ----------------------------------------------------------------------------------------------
def _global_model(tkg, pool=1, dropout=0.0, seed=0):
    from renet_b200.global_model import RENet_global
    torch.manual_seed(seed)
    return RENet_global(tkg.num_e, 200, tkg.num_r, dropout=dropout, model=3, seq_len=10, num_k=10, maxpool=pool).to(DEV)


def _predict_loop(m, t_list, graph_dict):
    """The per-timestamp definition (reference global_model.py:57-73)."""
    times = list(graph_dict.keys())
    unit = times[1] - times[0]
    out, prev = {}, 0
    for t in t_list:
        if t == 0:
            continue
        out[prev] = m.predict(t, graph_dict)[0].detach()
        prev = t
    out[t_list[-1]] = m.predict(t_list[-1] + unit, graph_dict)[0].detach()
    return out


def _assert_tables_equal(got, want, tol=1e-4):
    assert list(got) == list(want)
    for k in want:
        assert got[k].shape == (1, 1, 200) and not got[k].requires_grad
        a, r = got[k].view(-1).double().cpu(), want[k].view(-1).double().cpu()
        assert float((a - r).abs().max()) <= tol * max(1.0, float(r.abs().max())), k


def _tiny():
    from renet_b200 import synthetic
    return synthetic.SyntheticTKG('tiny', seed=7, num_timestamps=30)


@gpu
@pytest.mark.parametrize('pool', [1, 0])
def test_batched_table_equals_predict_loop(pool):
    tkg = _tiny()
    m = _global_model(tkg, pool).eval()
    t_list = sorted(tkg.graph_dict)
    with torch.no_grad():
        want = _predict_loop(m, t_list, tkg.graph_dict)
    _assert_tables_equal(m.get_global_emb(t_list, tkg.graph_dict), want)


@gpu
def test_batched_table_irregular_and_unsorted_keys_and_chunks(monkeypatch):
    from renet_b200 import global_model
    tkg = _tiny()
    m = _global_model(tkg).eval()
    keys = sorted(tkg.graph_dict)
    # irregular gaps: timestamps dropped from the stream (the windows follow the keys, not t // time unit)
    gaps = {t: tkg.graph_dict[t] for i, t in enumerate(keys) if i not in (3, 4, 9, 15, 16, 17, 22)}
    # keys out of order (the first one stays first, so no window is empty)
    order = keys[:5] + keys[5:12][::-1] + keys[12:20] + [keys[21], keys[20]] + keys[22:]
    unsorted = {t: tkg.graph_dict[t] for t in order}
    for gd in (gaps, unsorted):
        t_list = sorted(gd)
        with torch.no_grad():
            want = _predict_loop(m, t_list, gd)
        _assert_tables_equal(m.get_global_emb(t_list, gd), want)
    # a node budget of about three graphs: many chunks
    t_list = sorted(tkg.graph_dict)
    with torch.no_grad():
        want = _predict_loop(m, t_list, tkg.graph_dict)
    per_graph = max(g.number_of_nodes() for g in tkg.graph_dict.values())
    monkeypatch.setattr(global_model, 'GLOBAL_EMB_NODE_BUDGET', 3 * per_graph)
    _assert_tables_equal(m.get_global_emb(t_list, tkg.graph_dict), want)


@gpu
def test_batched_table_empty_window_and_train_mode():
    tkg = _tiny()
    keys = sorted(tkg.graph_dict)
    m = _global_model(tkg, dropout=0.5)
    no_zero = {t: tkg.graph_dict[t] for t in keys[1:]}         # t = keys[1] has no graph before it
    with pytest.raises(ValueError):
        m.get_global_emb(keys[1:], no_zero)
    m.eval()
    ev = m.get_global_emb(keys, tkg.graph_dict)
    m.train()
    torch.manual_seed(3)
    tr = m.get_global_emb(keys, tkg.graph_dict)
    assert list(tr) == list(ev)
    a = torch.cat([tr[k].view(-1) for k in tr])
    b = torch.cat([ev[k].view(-1) for k in ev])
    assert bool(torch.isfinite(a).all()) and float((a - b).abs().max()) > 1e-3


# ---- the pre-training step -------------------------------------------------------------------------------------------
def true_distribution(quads, num_e):
    """Restatement of the reference's get_true_distribution (utils.py:292-324), quirks included: a triple is counted
    before the timestamp change is detected, so each timestamp's first triple lands in the previous row, and the last
    row is not normalised."""
    rows_s, rows_o = [], []
    cur_s, cur_o = np.zeros(num_e), np.zeros(num_e)
    current_t = 0
    for s, _, o, t in np.asarray(quads, dtype=np.int64).tolist():
        cur_s[s] += 1
        cur_o[o] += 1
        if t != current_t:
            rows_s.append(cur_s / cur_s.sum())
            rows_o.append(cur_o / cur_o.sum())
            cur_s, cur_o = np.zeros(num_e), np.zeros(num_e)
            current_t = t
    rows_s.append(cur_s)
    rows_o.append(cur_o)
    return np.stack(rows_s), np.stack(rows_o)


STEP_SCRIPT = '''
import os, sys, torch
sys.path.insert(0, %r)
sys.path.insert(0, %r)
assert 'CUBLAS_WORKSPACE_CONFIG' not in os.environ
torch.use_deterministic_algorithms(True)
from test_gpu_global_pretrain import _tiny, _global_model, true_distribution
from renet_b200.parallel import DataParallelTrainer
tkg = _tiny()
times = sorted(tkg.graph_dict)
ps, po = (torch.from_numpy(a).cuda() for a in true_distribution(tkg.quads, tkg.num_e))
runs = []
for _ in range(2):
    m = _global_model(tkg, dropout=0.5).train()
    tr = DataParallelTrainer(m, lr=1e-3, weight_decay=1e-5, grad_norm=1.0)
    torch.manual_seed(1)
    for sel in ([5, 0, 17, 29, 3, 11], [2, 28, 14, 9]):
        tb = torch.tensor([times[i] for i in sel], device='cuda')
        tr.step(lambda: m(tb, ps[sel], po[sel], tkg.graph_dict), local_weight=len(sel))
        tr.zero_grad()
    torch.cuda.synchronize()
    runs.append([p.detach().cpu().clone() for p in m.parameters()])
assert all(torch.equal(a, b) for a, b in zip(*runs)), 'pre-training steps not bitwise reproducible'
print('PRETRAIN_DET_OK')
'''


@gpu
def test_pretrain_steps_need_no_cublas_and_are_bitwise_reproducible():
    env = {k: v for k, v in os.environ.items() if k != 'CUBLAS_WORKSPACE_CONFIG'}
    r = subprocess.run([sys.executable, '-c', STEP_SCRIPT % (ROOT, os.path.join(ROOT, 'tests'))], capture_output=True, text=True,
                       timeout=900, env=env, cwd=ROOT)
    sys.stdout.write(r.stdout)
    sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0 and 'PRETRAIN_DET_OK' in r.stdout


@pytest.mark.parametrize('pattern', [r'umma_gemm_packed_kernel<\(bool\)0, \(int\)3>', r'umma_gemm_packed_kernel<\(bool\)0, \(int\)4>',
                                     r'soft_ce_reduce_kernel\(', r'rowsum_accum_kernel\('])
def test_soft_ce_kernels_have_no_float_atomics(sass, pattern):
    found = {n: body for n, body in sass.items() if re.search(pattern, n)}
    assert found, 'no kernel matches %r' % pattern
    for name, body in found.items():
        hits = [ln.strip() for ln in body.split('\n') if FLOAT_ATOMIC.search(ln)]
        assert not hits, '%s: %s' % (name, hits[:3])


def _grads_of_one_step(m, t_sel, ps, po, gd, times, local_weight=None):
    from renet_b200.parallel import DataParallelTrainer
    tr = DataParallelTrainer(m, optimizer_step=lambda tr: None)
    tb = torch.tensor([times[i] for i in t_sel], device=ps.device)
    tr.step(lambda: m(tb, ps[t_sel], po[t_sel], gd), local_weight=local_weight)
    torch.cuda.synchronize()
    return {k: p.grad.detach().cpu().clone() for k, p in m.named_parameters()}


BATCH = [5, 0, 17, 29, 3, 11, 22, 8, 26, 14]


def _dp_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    from renet_b200.parallel import shard_slice
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    tkg = _tiny()
    times = sorted(tkg.graph_dict)
    ps, po = (torch.from_numpy(a).to(dev) for a in true_distribution(tkg.quads, tkg.num_e))
    lo, hi = shard_slice(len(BATCH), rank, world)
    m = _global_model(tkg).to(dev).train()
    grads = _grads_of_one_step(m, BATCH[lo:hi], ps, po, tkg.graph_dict, times, local_weight=hi - lo)
    torch.save(grads, os.path.join(out_dir, 'rank%d.pt' % rank))
    dist.barrier()
    dist.destroy_process_group()


@gpu
def test_pretrain_step_nccl_two_ranks_equals_single_process(tmp_path):
    """Each rank takes half of the timestamps, weighted by its count: the averaged gradients are the full batch's."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(('127.0.0.1', 0)); port = s.getsockname()[1]; s.close()
    mp.spawn(_dp_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    tkg = _tiny()
    times = sorted(tkg.graph_dict)
    ps, po = (torch.from_numpy(a).to(DEV) for a in true_distribution(tkg.quads, tkg.num_e))
    ref = _grads_of_one_step(_global_model(tkg).train(), BATCH, ps, po, tkg.graph_dict, times)
    for r in range(2):
        got = torch.load(os.path.join(str(tmp_path), 'rank%d.pt' % r))
        for k, g in ref.items():
            scale = float(g.abs().max()) + 1e-12
            assert float((got[k] - g).abs().max()) < 1e-5 * scale + 1e-9, (r, k)
