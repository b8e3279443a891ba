"""-m "not gpu": RENet.evaluate_stream_batched(process_group=...) with the model on the host, over gloo at world sizes 2 and 3.  Each
rank returns what the single-process call returns, and ends in the state it leaves (RNG included), bit for bit, on the
golden stream of renet_eval_tiny.npz with the CPU oracle standing in for the CUDA encode; ranks that disagree raise on every
rank instead of hanging."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from renet_b200 import parallel
from test_eval_batched_host import _assert_same_state, _ctx, _state

WORLD = 2
CASES = {'raw': dict(raw=True), 'filtered': dict(), 'time_aware': dict(time_aware=True)}


def _free_port():
    s = socket.socket(); s.bind(('127.0.0.1', 0)); p = s.getsockname()[1]; s.close()
    return p


def _stream(ctx):
    """The last validation timestamp, then the test split: three timestamps, two roll-overs."""
    quads, ev = ctx['quads'], ctx['ev']
    va_last = ev['va'][quads[ev['va'], 3] == quads[ev['va'], 3].max()]
    return np.concatenate((va_last[:8], ev['te']))


def _run(ctx, case, te=None, seed=1234, group=None):
    m, quads, gm = ctx['model'], ctx['quads'], ctx['gm']
    S, ST, O, OT = ctx['hist']
    te = _stream(ctx) if te is None else te
    kw = CASES[case]
    m.latest_time = torch.tensor(int(quads[te[0], 3]))
    torch.manual_seed(seed)
    return m.evaluate_stream_batched(quads[te], ([S[i] for i in te], [ST[i] for i in te]), ([O[i] for i in te], [OT[i] for i in te]),
                                     gm, total_data=None if kw.get('raw') else quads, process_group=group, **kw)


def _init(rank, port, world=WORLD):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)


def _sharded_worker(rank, port, out):
    _init(rank, port)
    try:
        for case in CASES:
            for rebinding in (True, False):
                ctx = _ctx(rebinding)
                got = _run(ctx, case, group=dist.group.WORLD)
                out[(case, rebinding, rank)] = (got, _state(ctx))
    finally:
        dist.destroy_process_group()


@pytest.fixture(scope='module')
def sharded():
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_sharded_worker, args=(_free_port(), out), nprocs=WORLD, join=True)
    res = dict(out)
    mgr.shutdown()
    return res


def _assert_same_result(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        if k == 'ranks':
            assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), k
        elif k == 'protocols':
            for p in a[k]:
                _assert_same_result(a[k][p], b[k][p])
        else:
            assert a[k] == b[k], k


@pytest.mark.parametrize('rebinding', [True, False])
@pytest.mark.parametrize('case', list(CASES))
def test_sharded_equals_single_process(sharded, case, rebinding):
    ctx = _ctx(rebinding)
    ref = _run(ctx, case)
    ref_state = _state(ctx)
    for rank in range(WORLD):
        got, state = sharded[(case, rebinding, rank)]
        _assert_same_result(got, ref)
        _assert_same_state(state, ref_state)


def test_chunks_go_to_exactly_one_rank():
    for n in (0, 1, 3, 7, 24):
        for world in range(1, 9):
            owned = [c for r in range(world) for c in parallel.round_robin(n, r, world)]
            assert sorted(owned) == list(range(n)), (n, world)
            for r in range(world):
                assert all(c % world == r for c in parallel.round_robin(n, r, world))


def _mismatch_worker(rank, port, out):
    _init(rank, port)
    try:
        one = dist.new_group([0])                 # every rank takes part in creating it; only rank 0 is in it
        ctx = _ctx()
        te = _stream(ctx)
        res = {}
        try:
            ctx['model']._eval_shard(one)
            res['not_member'] = None
        except ValueError as e:
            res['not_member'] = str(e)
        res['size_one'] = ctx['model']._eval_shard(one) is None if rank == 0 else None
        try:                                      # rank 1 drops its last test triple
            _run(ctx, 'filtered', te=te if rank == 0 else te[:-1], group=dist.group.WORLD)
            res['fingerprint'] = None
        except ValueError as e:
            res['fingerprint'] = str(e)
        try:                                      # the same arguments, different seeds: the first roll-over's picks differ
            _run(ctx, 'filtered', te=te, seed=1234 + rank, group=dist.group.WORLD)
            res['picks'] = None
        except RuntimeError as e:
            res['picks'] = str(e)
        out[rank] = res
    finally:
        dist.destroy_process_group()


def test_ranks_that_disagree_raise_on_every_rank():
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_mismatch_worker, args=(_free_port(), out), nprocs=WORLD, join=True)
    res = dict(out)
    mgr.shutdown()
    assert res[0]['not_member'] is None and res[0]['size_one'] is True
    assert 'not a member' in res[1]['not_member']
    for rank in range(WORLD):
        assert 'different test data' in res[rank]['fingerprint'], res[rank]
        assert 'different roll-over picks' in res[rank]['picks'], res[rank]


def _one_triple_stream(ctx):
    """A timestamp of ONE triple (2 rank rows), then the test split after a roll-over."""
    quads, ev = ctx['quads'], ctx['ev']
    va_last = ev['va'][quads[ev['va'], 3] == quads[ev['va'], 3].max()]
    return np.concatenate((va_last[:1], ev['te']))


def _few_rows_worker(rank, port, out):
    _init(rank, port, world=3)
    try:
        ctx = _ctx()
        got = _run(ctx, 'time_aware', te=_one_triple_stream(ctx), group=dist.group.WORLD)
        out[rank] = (got, _state(ctx))
    finally:
        dist.destroy_process_group()


def test_ranks_without_rows_take_part():
    """World size 3 over a timestamp of 2 rank rows: one rank ranks no row and still takes part in every exchange."""
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_few_rows_worker, args=(_free_port(), out), nprocs=3, join=True)
    res = dict(out)
    mgr.shutdown()
    ctx = _ctx()
    te = _one_triple_stream(ctx)
    assert np.sum(ctx['quads'][te, 3] == ctx['quads'][te[0], 3]) == 1
    ref = _run(ctx, 'time_aware', te=te)
    ref_state = _state(ctx)
    for rank in range(3):
        got, state = res[rank]
        _assert_same_result(got, ref)
        _assert_same_state(state, ref_state)
