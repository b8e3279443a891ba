"""-m gpu: RENet.evaluate_stream_batched(process_group=...) on the kernels over NCCL, one process per GPU, and over gloo with
both ranks on one GPU (the exchanges through the host; this runs on a machine with one GPU).  At world size 2
every rank returns the single-process result and ends in the single-process state, torch's CPU and CUDA RNG included, bit
for bit: on the ICEWS18-shaped stream of test_gpu_eval_batched.py (three test timestamps, two roll-overs, time-aware
protocols) and on the golden run of renet_eval_global.npz with both models on the kernels.  A group of one runs unsharded."""
import hashlib
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from helpers import load_npz

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket(); s.bind(('127.0.0.1', 0)); p = s.getsockname()[1]; s.close()
    return p


def _digest(m, gm_calls):
    """A hash of the evaluation state: histories, caches, graph_dict, global_emb, latest_time and the global model's calls."""
    h = hashlib.blake2b(digest_size=16)
    for name in ('s_hist_test', 'o_hist_test', 's_his_cache', 'o_his_cache'):
        for x in getattr(m, name):
            for a in (x if isinstance(x, list) else [x]):
                a = np.asarray(torch.as_tensor(a).cpu(), dtype=np.int64)
                h.update(repr(a.shape).encode()); h.update(a.tobytes())
            h.update(b'|')
    for name in ('s_hist_test_t', 'o_hist_test_t', 's_his_cache_t', 'o_his_cache_t'):
        h.update(repr([list(map(int, x)) if isinstance(x, list) else x for x in getattr(m, name)]).encode())
    for t in sorted(m.graph_dict):
        g = m.graph_dict[t]
        h.update(repr((int(t), g.number_of_edges())).encode()); h.update(g.ndata['id'].cpu().numpy().tobytes())
    for t in sorted(m.global_emb):
        h.update(repr(int(t)).encode()); h.update(m.global_emb[t].detach().cpu().numpy().tobytes())
    h.update(repr((int(m.latest_time), gm_calls)).encode())
    return h.hexdigest()


def _icews18(group=None):
    from test_gpu_eval_batched import _icews18_stream
    quads, te, (S, ST, O, OT), ((m, gm), _) = _icews18_stream()
    torch.manual_seed(77)
    out = m.evaluate_stream_batched(quads[te], ([S[i] for i in te], [ST[i] for i in te]), ([O[i] for i in te], [OT[i] for i in te]),
                                    gm, total_data=quads, time_aware=True, process_group=group)
    return dict(out=out, rng=(torch.get_rng_state(), torch.cuda.get_rng_state()), state=_digest(m, gm.calls))


def _global(group=None):
    """The golden run of renet_eval_global.npz (the reference's global model) with both models on the kernels, set up as
    test_gpu_eval_batched.test_batched_flow_with_the_global_model_matches_reference_golden sets it up."""
    from oracle import restate
    from oracle.gen_golden import RENET_SHAPES, det_params
    from renet_b200 import synthetic
    from renet_b200.global_model import RENet_global
    from renet_b200.model import RENet
    from test_gpu_eval_global import _HostOutputs
    ev, tiny = load_npz('renet_eval_global.npz'), load_npz('renet_tiny.npz')
    quads = tiny['quads'].astype(np.int64)
    num_e, R, h, nb, seed, num_k = int(tiny['num_e']), int(tiny['R']), int(ev['h']), int(ev['nb']), int(ev['seed']), int(ev['num_k'])
    gshapes = {str(k): tuple(int(x) for x in v[:2] if x > 0) for k, v in zip(ev['gshape_keys'], ev['gshape_vals'])}
    gm = RENet_global(num_e, h, R, dropout=0, model=3, seq_len=10, num_k=num_k, maxpool=1)
    gm.load_state_dict(det_params(gshapes, seed + 1), strict=True)
    gm = gm.cuda().eval()
    m = RENet(num_e, h, R, dropout=0, model=0, seq_len=10, num_k=num_k, num_bases=nb)
    m.load_state_dict(det_params(RENET_SHAPES(num_e, h, R, nb), seed), strict=True)
    m = m.cuda().eval()
    gd = synthetic.build_graph_dict(quads, R)
    tr, va, te = ev['tr'], ev['va'], ev['te']
    with torch.no_grad():
        m.global_emb = gm.get_global_emb([int(t) for t in np.unique(quads[tr][:, 3])], gd)
    m.graph_dict = gd
    S, ST, O, OT = restate.build_history(quads, num_e)
    pick = lambda L, idx: [L[i] for i in idx]                                           # noqa: E731
    m.init_history(quads[tr], (pick(S, tr), pick(ST, tr)), (pick(O, tr), pick(OT, tr)),
                   quads[va], (pick(S, va), pick(ST, va)), (pick(O, va), pick(OT, va)),
                   quads[te], (pick(S, te), pick(ST, te)), (pick(O, te), pick(OT, te)))
    m.latest_time = torch.tensor(int(quads[te[0], 3]))
    torch.manual_seed(4321)
    out = m.evaluate_stream_batched(quads[te], (pick(S, te), pick(ST, te)), (pick(O, te), pick(OT, te)), _HostOutputs(gm),
                                    total_data=quads, process_group=group)
    return dict(out=out, rng=(torch.get_rng_state(), torch.cuda.get_rng_state()), state=_digest(m, []))


def _init(rank, world, port, backend='nccl'):
    """NCCL: rank r owns GPU r.  gloo: every rank runs on GPU 0 and the exchanges go through the host, which checks the
    sharding of the kernel path on a machine with one GPU."""
    if backend == 'nccl':
        os.environ['CUDA_VISIBLE_DEVICES'] = str(rank)      # before CUDA starts in this process
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(0)
    if backend == 'nccl':
        dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', 0))
    else:
        dist.init_process_group('gloo', rank=rank, world_size=world)


def _sharded_worker(rank, world, port, backend, out):
    _init(rank, world, port, backend)
    try:
        res = {'icews18': _icews18(dist.group.WORLD), 'global': _global(dist.group.WORLD)}
        if backend == 'nccl':                               # a model on the host cannot take an NCCL group
            from helpers import eval_setup
            ctx = eval_setup('cpu')
            try:
                ctx['model'].evaluate_stream_batched(ctx['quads'][:4], ([[]] * 4, [[]] * 4), ([[]] * 4, [[]] * 4), ctx['gm'],
                                                     raw=True, process_group=dist.group.WORLD)
                res['host_on_nccl'] = None
            except ValueError as e:
                res['host_on_nccl'] = str(e)
        out[rank] = res
    finally:
        dist.destroy_process_group()


def _single_worker(rank, world, port, backend, out):
    _init(rank, world, port)
    try:
        from renet_b200 import parallel

        def no_shard(*a, **kw):
            raise AssertionError('a group of one must run unsharded')
        parallel.Shard = no_shard
        out[rank] = _global(dist.group.WORLD)
    finally:
        dist.destroy_process_group()


def _spawn(fn, world, backend='nccl'):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(fn, args=(world, _free_port(), backend, out), nprocs=world, join=True)
    res = dict(out)
    mgr.shutdown()
    return res


def _assert_same(got, ref):
    a, b = got['out'], ref['out']
    assert sorted(a) == sorted(b)
    for k in a:
        if k == 'ranks':
            assert np.array_equal(a[k], b[k]), k
        elif k == 'protocols':
            for p in a[k]:
                assert np.array_equal(a[k][p]['ranks'], b[k][p]['ranks']), p
                assert all(a[k][p][q] == b[k][p][q] for q in a[k][p] if q != 'ranks'), p
        else:
            assert a[k] == b[k], k
    assert torch.equal(got['rng'][0], ref['rng'][0]) and torch.equal(got['rng'][1], ref['rng'][1])
    assert got['state'] == ref['state']


@pytest.mark.parametrize('backend', ['nccl', 'gloo'])
def test_sharded_evaluation_equals_single_process_bitwise(backend):
    if backend == 'nccl' and torch.cuda.device_count() < 2:
        pytest.skip('NCCL at world size 2 needs 2 GPUs')
    res = _spawn(_sharded_worker, 2, backend)
    ref_icews, ref_global = _icews18(), _global()
    for rank in range(2):
        _assert_same(res[rank]['icews18'], ref_icews)
        _assert_same(res[rank]['global'], ref_global)
        if backend == 'nccl':
            assert 'needs the model on a GPU' in res[rank]['host_on_nccl']
    assert len(ref_icews['out']['protocols']['time_filtered']['ranks']) > 1000
    ev = load_npz('renet_eval_global.npz')                # and the single-process run is the golden's
    out = ref_global['out']
    assert abs(out['mrr'] - float(ev['mrr'])) < 5e-4 and np.mean(out['ranks'] == ev['ranks']) > 0.98


def test_group_of_one_runs_unsharded():
    res = _spawn(_single_worker, 1)
    _assert_same(res[0], _global())


# ---- more ranks than rows --------------------------------------------------------------------------------------------------
def _tiny(group=None):
    """The golden stream of renet_eval_tiny.npz on the kernels, starting with a timestamp of ONE triple (2 rank rows), then
    the test split after a roll-over; time-aware, so every rank call takes two exclusion lists."""
    from helpers import eval_setup
    ctx = eval_setup('cuda')
    m, quads, gm, ev = ctx['model'], ctx['quads'], ctx['gm'], ctx['ev']
    S, ST, O, OT = ctx['hist']
    va_last = ev['va'][quads[ev['va'], 3] == quads[ev['va'], 3].max()]
    te = np.concatenate((va_last[:1], ev['te']))
    assert np.sum(quads[te, 3] == quads[te[0], 3]) == 1
    m.latest_time = torch.tensor(int(quads[te[0], 3]))
    torch.manual_seed(1234)
    out = m.evaluate_stream_batched(quads[te], ([S[i] for i in te], [ST[i] for i in te]), ([O[i] for i in te], [OT[i] for i in te]),
                                    gm, total_data=quads, time_aware=True, process_group=group)
    return dict(out=out, rng=(torch.get_rng_state(), torch.cuda.get_rng_state()), state=_digest(m, gm.calls))


def _tiny_worker(rank, world, port, backend, out):
    _init(rank, world, port, backend)
    try:
        out[rank] = _tiny(dist.group.WORLD)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('backend', ['nccl', 'gloo'])
def test_ranks_without_rows_take_part(backend):
    """World size 3 over a timestamp of 2 rank rows: one rank ranks no row and must still take part in every exchange."""
    if backend == 'nccl' and torch.cuda.device_count() < 3:
        pytest.skip('NCCL at world size 3 needs 3 GPUs')
    res = _spawn(_tiny_worker, 3, backend)
    ref = _tiny()
    for rank in range(3):
        _assert_same(res[rank], ref)


def test_rank_rows_without_rows_launch_nothing():
    """_rank_rows on zero rows: no launch, and the dtypes and widths of a call with rows, for 0-2 exclusion lists."""
    from helpers import eval_setup
    from renet_b200 import _lib
    m = eval_setup('cuda')['model']
    K = m.linear.weight.shape[1]
    x = torch.randn(3, K, device='cuda')
    empty = np.zeros(0, np.int64)
    for n_lists in (0, 1, 2):
        ex_full = [(np.asarray([1, 2], np.int32), np.asarray([0, 1, 2]), np.asarray([1, 2, 2]))] * n_lists
        ex_none = [(np.asarray([1, 2], np.int32), empty, empty)] * n_lists
        with torch.no_grad():
            l3, c3 = m._rank_rows(x, np.asarray([0, 1, 2]), ex_full)
            n0 = _lib.launch_count()
            l0, c0 = m._rank_rows(x[:0], empty, ex_none)
        assert _lib.launch_count() == n0
        assert l0.shape == (0,) and c0.shape == (0, 2 + 2 * n_lists)
        assert (l0.dtype, l0.device, c0.dtype, c0.device) == (l3.dtype, l3.device, c3.dtype, c3.device)
