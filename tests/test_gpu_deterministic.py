"""-m gpu: deterministic mode.  Under torch.use_deterministic_algorithms(True) every backward entry point returns bitwise
identical results on identical inputs and stays within the usual tolerances of float64; a whole training step, repeated
from the same seeds, gives bitwise identical parameters; the switch follows torch's flag both ways."""
import contextlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gpu_helpers import DEV, layer_bwd
from oracle import restate

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUNS = 3


@contextlib.contextmanager
def deterministic():
    from renet_b200 import _lib
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        _lib.stream()
        assert _lib.lib().renet_get_deterministic() == 1
        yield
    finally:
        torch.use_deterministic_algorithms(before)
        _lib.stream()


def assert_runs_equal(runs):
    for k in runs[0]:
        for r in runs[1:]:
            assert torch.equal(runs[0][k], r[k]), k


def rel(got, ref):
    return float((got.double().cpu() - ref).abs().max() / ref.abs().max())


def test_switch_follows_torch_flag():
    from renet_b200 import _lib
    L = _lib.lib()
    assert not torch.are_deterministic_algorithms_enabled()
    _lib.stream()
    assert L.renet_get_deterministic() == 0
    with deterministic():
        assert L.renet_get_deterministic() == 1
    assert L.renet_get_deterministic() == 0
    assert L.renet_set_deterministic(1) == 0 and L.renet_set_deterministic(0) == 1


# ---- RGCN layer backward ------------------------------------------------------------------------------------------------
def _graph(N, E, R2, seed, hub_rel_share=0.3, hub_src_share=0.05, N_dst=None):
    """ICEWS18-like skew: one relation carries hub_rel_share of the edges, one source entity hub_src_share."""
    rng = np.random.RandomState(seed)
    N_dst = N if N_dst is None else N_dst
    src = rng.randint(0, N, E)
    src[rng.rand(E) < hub_src_share] = 7
    dst = rng.randint(0, N_dst, E)
    et = rng.randint(0, R2, E)
    et[rng.rand(E) < hub_rel_share] = 3
    deg = np.bincount(dst, minlength=N).astype(np.float32)
    norm = (1.0 / np.maximum(deg, 1)).astype(np.float32)
    return src, dst, et, norm


def _layer_case(N, E, indexed, seed):
    R2, h = 460, 200
    src, dst, et, norm = _graph(N, E, R2, seed)
    g = torch.Generator(device=DEV).manual_seed(seed)
    table = torch.randn(23033 if indexed else N, h, device=DEV, generator=g) * 0.5
    h_index = torch.randint(0, table.shape[0], (N,), device=DEV, generator=g, dtype=torch.int32) if indexed else None
    W = torch.randn(R2, 400, device=DEV, generator=g) * 0.3
    Wloop = torch.randn(h, h, device=DEV, generator=g) * 0.07
    dout = torch.randn(N, h, device=DEV, generator=g)
    Hin = table[h_index.long()] if indexed else table
    s64, d64, t64 = (torch.from_numpy(x.astype(np.int64)) for x in (src, dst, et))
    leaves = [Hin.double().cpu().requires_grad_(True), W.double().cpu().requires_grad_(True),
              Wloop.double().cpu().requires_grad_(True)]
    out = restate.rgcn_block_layer(*leaves, s64, d64, t64, torch.from_numpy(norm).double(), True, 100)
    (out * dout.double().cpu()).sum().backward()
    Hout = out.detach().float().to(DEV)
    ref = {'dH': leaves[0].grad, 'dW': leaves[1].grad, 'dWloop': leaves[2].grad}

    def run():
        dH, dW, dWl = layer_bwd(table, h_index, W, Wloop, src, dst, et, torch.from_numpy(norm).to(DEV), Hout, dout, N, E,
                                h, h, 100, True)
        return {'dH': dH, 'dW': dW, 'dWloop': dWl}
    return run, ref


@pytest.mark.parametrize('N,E,indexed', [(30000, 120000, True),     # stream kernel for dH (16 k <= N <= 40 k, E >= 16 k)
                                         (3000, 12000, False)])     # tile kernel for dH
def test_rgcn_block_bwd(N, E, indexed):
    run, ref = _layer_case(N, E, indexed, seed=N)
    with deterministic():
        runs = [run() for _ in range(RUNS)]
    assert_runs_equal(runs)
    for k in ref:
        assert rel(runs[0][k], ref[k]) < 1e-4, k


def test_rgcn_bipartite_bwd():
    from renet_b200 import _lib
    from renet_b200.graph import build_csr
    L = _lib.lib()
    N_src, N_dst, E, R2, h = 6000, 2500, 20000, 460, 200
    src, dst, et, norm = _graph(N_src, E, R2, 5, N_dst=N_dst)
    g = torch.Generator(device=DEV).manual_seed(5)
    H = torch.randn(N_src, h, device=DEV, generator=g) * 0.5
    W = torch.randn(R2, 400, device=DEV, generator=g) * 0.3
    dout = torch.randn(N_dst, h, device=DEV, generator=g)
    Hd, Wd = H.double().cpu().requires_grad_(True), W.double().cpu().requires_grad_(True)
    s64, d64, t64 = (torch.from_numpy(x.astype(np.int64)) for x in (src, dst, et))
    out = restate.rgcn_block_layer(Hd, Wd, None, s64, d64, t64, torch.from_numpy(norm).double(), False, 100)[:N_dst]
    (out * dout.double().cpu()).sum().backward()
    i32 = lambda x: torch.from_numpy(x.astype(np.int32)).to(DEV)
    t_rp, t_cd, t_ct, _ = build_csr(i32(src), i32(dst), i32(et), N_src)
    r_rp, r_src, r_dst, _ = build_csr(i32(et), i32(src), i32(dst), R2)
    normd = torch.from_numpy(norm[:N_dst]).to(DEV)
    base = torch.randn(R2, 400, device=DEV, generator=g) * 1e-2
    ws = torch.empty(((N_dst * h + 3) // 4) * 4 + h * h, device=DEV)
    P = _lib.ptr

    def run():
        dH, dW = torch.full((N_src, h), float('nan'), device=DEV), base.clone()
        _lib.check(L.renet_rgcn_bipartite_bwd(P(H), P(W), P(t_rp), P(t_cd), P(t_ct), P(r_rp), P(r_src), P(r_dst), P(normd), None,
                                              P(dout), P(dH), P(dW), P(ws), N_src, N_dst, E, h, h, 100, R2, 0, _lib.stream()),
                   'renet_rgcn_bipartite_bwd')
        return {'dH': dH, 'dW': dW.double() - base.double()}
    with deterministic():
        runs = [run() for _ in range(RUNS)]
    assert_runs_equal(runs)
    assert rel(runs[0]['dH'], Hd.grad) < 1e-4 and rel(runs[0]['dW'], Wd.grad) < 1e-4


def test_selfloop_gemm_bwd_indexed():
    from renet_b200 import _lib
    L, P = _lib.lib(), _lib.ptr
    N, h = 34500, 200
    g = torch.Generator(device=DEV).manual_seed(11)
    table = torch.randn(23033, h, device=DEV, generator=g)
    idx = torch.randint(0, 23033, (N,), device=DEV, generator=g, dtype=torch.int32)
    Wloop = torch.randn(h, h, device=DEV, generator=g) * 0.07
    dLoop = torch.randn(N, h, device=DEV, generator=g)
    base = torch.randn(h, h, device=DEV, generator=g)
    ws = torch.empty(h * h, device=DEV)

    def run():
        dH, dWl = torch.full((N, h), float('nan'), device=DEV), base.clone()
        _lib.check(L.renet_selfloop_gemm_bwd(P(table), P(idx), P(Wloop), P(dLoop), P(dH), P(dWl), P(ws), N, h, h, _lib.stream()),
                   'renet_selfloop_gemm_bwd')
        return {'dH': dH, 'dWloop': dWl.double() - base.double()}
    with deterministic():
        runs = [run() for _ in range(RUNS)]
    assert_runs_equal(runs)
    Hin, dL = table[idx.long()].double(), dLoop.double()
    assert rel(runs[0]['dH'], (dL @ Wloop.double().t()).cpu()) < 1e-5
    assert rel(runs[0]['dWloop'], (Hin.t() @ dL).cpu()) < 1e-5


def test_scatter_add_rows_hub_target_unaligned_width():
    from renet_b200 import _lib
    L, P = _lib.lib(), _lib.ptr
    n, d, T = 30000, 203, 500                      # d % 4 != 0: the scalar kernel's ground in the atomic mode
    g = torch.Generator(device=DEV).manual_seed(3)
    idx = torch.randint(0, T, (n,), device=DEV, generator=g, dtype=torch.int32)
    idx[torch.randperm(n, device=DEV, generator=g)[:10000]] = 42      # one target receives 10 k rows
    src = torch.randn(n, d, device=DEV, generator=g)
    base = torch.randn(T, d, device=DEV, generator=g)

    def run():
        dst = base.clone()
        _lib.check(L.renet_scatter_add_rows(P(src), P(idx), P(dst), n, d, _lib.stream()), 'renet_scatter_add_rows')
        return {'dst': dst}
    with deterministic():
        runs = [run() for _ in range(RUNS)]
    assert_runs_equal(runs)
    ref = torch.zeros(T, d, dtype=torch.float64, device=DEV).index_add_(0, idx.long(), src.double())
    assert rel(runs[0]['dst'].double() - base.double(), ref.cpu()) < 1e-5


# ---- GRU backward entry points ------------------------------------------------------------------------------------------
def _gru_case(kind):
    """run(): the forward and renet_gru_bwd / renet_gru_bwd_dropout (p = 0.5) / renet_gru_dense_bwd on fixed inputs."""
    from renet_b200 import _lib
    L, P = _lib.lib(), _lib.ptr
    h, T, num_e, num_r = 200, 37, 5000, 460
    lens = np.array([10] * 300 + [6] * 500 + [3] * 700 + [1] * 400, dtype=np.int64)
    Q, S, max_len = len(lens), int(lens.sum()), int(lens.max())
    bs = np.array([int((lens > t).sum()) for t in range(max_len)], dtype=np.int32)
    hbs = bs.ctypes.data_as(_lib.ctypes.c_void_p)
    g = torch.Generator(device=DEV).manual_seed(21)
    rnd = lambda *s, sc=1.0: torch.randn(*s, device=DEV, generator=g) * sc
    ri = lambda hi, n: torch.randint(0, hi, (n,), device=DEV, generator=g, dtype=torch.int32)
    NH = S // 2
    H2, ent, rel_, glob = rnd(NH, h, sc=0.5), rnd(num_e, h, sc=0.3), rnd(num_r, h, sc=0.3), rnd(T, h, sc=0.1)
    readout, row_glob, seq_s, seq_r = ri(NH, S), ri(T, S), ri(num_e, Q), ri(num_r, Q)
    row_seq = torch.from_numpy(np.repeat(np.arange(Q), lens).astype(np.int32)).to(DEV)
    seq_len = torch.from_numpy(lens.astype(np.int32)).to(DEV)
    seq_start = torch.from_numpy(np.concatenate(([0], np.cumsum(lens)[:-1])).astype(np.int32)).to(DEV)
    dense = kind == 'dense'
    k4 = h if dense else 4 * h
    sc = 1.0 / h ** 0.5
    W = [rnd(3 * h, k4, sc=sc), rnd(3 * h, h, sc=sc), rnd(3 * h, sc=0.1), rnd(3 * h, sc=0.1),
         rnd(3 * h, 3 * h, sc=sc), rnd(3 * h, h, sc=sc), rnd(3 * h, sc=0.1), rnd(3 * h, sc=0.1)]
    hn4, hn3, dhn4, dhn3 = rnd(Q, h), rnd(Q, h), rnd(Q, h), rnd(Q, h)
    stream, seed, p = _lib.stream(), 1234, 0.5
    X4 = rnd(S, k4, sc=0.5) if dense else None
    if dense:
        nbytes, bbytes = int(L.renet_gru_dropout_workspace_bytes(S, Q, 1, h)), int(L.renet_gru_bwd_dropout_workspace_bytes(S, Q, 1, h))
    elif kind == 'dropout':
        nbytes, bbytes = int(L.renet_gru_dropout_workspace_bytes(S, Q, T, h)), int(L.renet_gru_bwd_dropout_workspace_bytes(S, Q, T, h))
    else:
        nbytes, bbytes = int(L.renet_gru_workspace_bytes(S, Q, T, h)), int(L.renet_gru_bwd_workspace_bytes(S, Q, T, h))
    names = ['w_ih4', 'w_hh4', 'b_ih4', 'b_hh4'] + ([] if dense else ['w_ih3', 'w_hh3', 'b_ih3', 'b_hh3', 'd_ent', 'd_rel', 'd_glob'])
    shapes = {'d_ent': ent.shape, 'd_rel': rel_.shape, 'd_glob': glob.shape}
    bases = {k: rnd(*(shapes[k] if k in shapes else W[names.index(k)].shape)) for k in names}

    def run():
        # the backward consumes the forward's workspace: every run starts with its own forward
        ws, bws = torch.empty(nbytes // 4, device=DEV), torch.empty(bbytes // 4, device=DEV)
        wp = [P(t) for t in W]
        if dense:
            rc = L.renet_gru_dense_fwd(P(X4), k4, None, 0, P(seq_len), P(seq_start), hbs, max_len, *wp[:4], None, None, None, None,
                                       P(hn4), P(hn3), S, Q, h, P(ws), nbytes, stream)
        elif kind == 'dropout':
            rc = L.renet_gru_fwd_dropout(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel_), P(row_seq), P(seq_s), P(seq_r),
                                         P(seq_len), P(seq_start), hbs, max_len, *wp, P(hn4), P(hn3), S, Q, T, h, p, seed, P(ws), nbytes,
                                         stream)
        else:
            rc = L.renet_gru_fwd(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel_), P(seq_s), P(seq_r), P(seq_len), P(seq_start),
                                 hbs, max_len, *wp, P(hn4), P(hn3), S, Q, T, h, P(ws), nbytes, stream)
        _lib.check(rc, 'gru forward (%s)' % kind)
        acc = {k: v.clone() for k, v in bases.items()}
        dw = [P(acc.get(k)) for k in ('w_ih4', 'w_hh4', 'b_ih4', 'b_hh4', 'w_ih3', 'w_hh3', 'b_ih3', 'b_hh3')]
        wb = [wp[0], wp[1], wp[4], wp[5]]
        st = _lib.stream()
        if dense:
            acc['dX4'] = torch.full((S, k4), float('nan'), device=DEV)
            rc = L.renet_gru_dense_bwd(P(X4), k4, None, 0, P(seq_len), P(seq_start), hbs, max_len, wb[0], wb[1], None, None,
                                       P(dhn4), P(dhn3), P(acc['dX4']), None, *dw[:4], None, None, None, None, S, Q, h, P(ws),
                                       P(bws), bbytes, st)
        else:
            acc['dH2'] = torch.full((NH, h), float('nan'), device=DEV)
            common = (P(acc['dH2']), P(acc['d_ent']), P(acc['d_rel']), P(acc['d_glob']), *dw, NH, S, Q, T, h)
            if kind == 'dropout':
                rc = L.renet_gru_bwd_dropout(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel_), P(row_seq), P(seq_s),
                                             P(seq_r), P(seq_len), P(seq_start), hbs, max_len, *wb, P(dhn4), P(dhn3), *common, p,
                                             seed, P(ws), P(bws), bbytes, st)
            else:
                rc = L.renet_gru_bwd(P(H2), P(readout), P(row_glob), P(glob), P(ent), P(rel_), P(seq_s), P(seq_r), P(seq_len),
                                     P(seq_start), hbs, max_len, *wb, P(dhn4), P(dhn3), *common, P(ws), P(bws), bbytes, st)
        _lib.check(rc, 'gru backward (%s)' % kind)
        return acc
    return run


@pytest.mark.parametrize('kind', ['plain', 'dropout', 'dense'])
def test_gru_bwd(kind):
    run = _gru_case(kind)
    with deterministic():
        runs = [run() for _ in range(RUNS)]
    assert_runs_equal(runs)
    for k, v in runs[0].items():
        assert not torch.isnan(v).any(), k


def _contract_script_in_deterministic_mode(script, marker):
    """The fp64 contract checks of the GEMM engine and the GRU, run with torch's deterministic flag on (warn_only: the
    float64 references use torch ops of their own), so every library call in them takes the deterministic path."""
    code = ('import runpy, sys, torch\n'
            'torch.use_deterministic_algorithms(True, warn_only=True)\n'
            'from renet_b200 import _lib\n'
            '_lib.stream()\n'
            'assert _lib.lib().renet_get_deterministic() == 1\n'
            'sys.argv = [%r]\n'
            'runpy.run_path(%r, run_name="__main__")\n' % (script, script))
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=':4096:8')
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    sys.stdout.write(r.stdout)
    sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0 and marker in r.stdout


def test_gru_contract_in_deterministic_mode():
    _contract_script_in_deterministic_mode(os.path.join(ROOT, 'tests', 'gru_contract_check.py'), 'GRU_CONTRACT_OK')


def test_gemm_contract_in_deterministic_mode():
    _contract_script_in_deterministic_mode(os.path.join(ROOT, 'tests', 'gemm_contract_check.py'), 'GEMM_CONTRACT_OK')


# ---- whole training step ------------------------------------------------------------------------------------------------
def _train_params(dev, rank=0, world=1, steps=3):
    from renet_b200 import synthetic
    from renet_b200.model import RENet
    from renet_b200.parallel import DataParallelTrainer, shard_batch
    tkg = synthetic.SyntheticTKG('icews18', seed=17, num_timestamps=30)
    torch.manual_seed(0)
    m = RENet(tkg.num_e, 200, tkg.num_r, dropout=0.5).to(dev).train()
    m.global_emb = {t: v.to(dev) for t, v in tkg.global_emb.items()}
    tr = DataParallelTrainer(m, lr=1e-3, weight_decay=1e-5, grad_norm=1.0)
    for i in range(steps):
        q, sh, oh = tkg.batch(i, batch_size=1024 * world)
        if world > 1:
            q, sh, oh, _ = shard_batch(q, sh, oh, rank, world)
        tr.train_step(torch.from_numpy(q).to(dev), sh, oh, tkg.graph_dict)
    torch.cuda.synchronize()
    return {k: p.detach().clone().cpu() for k, p in m.named_parameters()}


def test_training_steps_bitwise_reproducible():
    with deterministic():
        a = _train_params(DEV)
        b = _train_params(DEV)
    assert_runs_equal([a, b])


def _dp_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    torch.use_deterministic_algorithms(True)
    runs = [_train_params(dev, rank, world) for _ in range(2)]
    torch.save(runs, os.path.join(out_dir, 'rank%d.pt' % rank))
    dist.barrier()
    dist.destroy_process_group()


def test_training_steps_bitwise_reproducible_nccl_two_ranks(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(('127.0.0.1', 0)); port = s.getsockname()[1]; s.close()
    mp.spawn(_dp_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    for r in range(2):
        assert_runs_equal(torch.load(os.path.join(str(tmp_path), 'rank%d.pt' % r)))


GLOBAL_SCRIPT = '''
import sys, torch
sys.path.insert(0, %r)
sys.path.insert(0, %r)
torch.use_deterministic_algorithms(True)
from helpers import global_setup
from renet_b200 import synthetic
from renet_b200.global_model import RENet_global
c = global_setup()
gd = synthetic.build_graph_dict(c['quads'], c['R'])
runs = []
for _ in range(2):
    m = RENet_global(c['num_e'], c['h'], c['R'], dropout=0, model=3, seq_len=10, num_k=10, maxpool=1)
    m.load_state_dict(c['params'], strict=True)
    m = m.to('cuda:0').train()
    tps = torch.from_numpy(c['tps'][c['sel']]).to('cuda:0')
    tpo = torch.from_numpy(c['tpo'][c['sel']]).to('cuda:0')
    loss = m(torch.from_numpy(c['t_batch']), tps, tpo, gd, subject=True)
    loss.backward()
    runs.append([loss.detach().cpu()] + [p.grad.detach().cpu() for p in m.parameters() if p.grad is not None])
assert len(runs[0]) > 5
assert all(torch.equal(a, b) for a, b in zip(*runs)), 'global model forward/backward not bitwise reproducible'
print('GLOBAL_DET_OK')
'''


def test_global_model_bitwise_reproducible():
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=':4096:8')
    r = subprocess.run([sys.executable, '-c', GLOBAL_SCRIPT % (ROOT, os.path.join(ROOT, 'tests'))], capture_output=True, text=True,
                       timeout=900, env=env, cwd=ROOT)
    sys.stdout.write(r.stdout)
    sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0 and 'GLOBAL_DET_OK' in r.stdout


def test_golden_gradient_parity_in_deterministic_mode():
    """The reference-golden gradient tests (renet_icews18_slice.npz, global_tiny.npz) pass with the switch on."""
    code = ('import sys, torch, pytest\n'
            'torch.use_deterministic_algorithms(True, warn_only=True)\n'
            'sys.exit(pytest.main(["-q", "-p", "no:cacheprovider", '
            '"tests/test_gpu_gru_renet.py::test_fused_training_step_gradients_match_reference_golden", '
            '"tests/test_gpu_global.py::test_global_forward_backward_matches_reference_golden"]))\n')
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=':4096:8')
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    sys.stdout.write(r.stdout[-3000:])
    sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0 and ' passed' in r.stdout and 'failed' not in r.stdout
