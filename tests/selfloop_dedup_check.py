"""Run in a subprocess by tests/test_gpu_selfloop_dedup.py: the deduplicated indexed self-loop product.

An indexed product of at least kDedupMinRows rows computes each distinct index once and copies the rows out.  For every
index pattern below, `renet_selfloop_gemm(A, idx)` must be bitwise equal to the plain product on the materialised A[idx],
leave the rows past M untouched, and take the path its size selects (counted in kernel launches)."""
import os
import re
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from renet_b200 import _lib  # noqa: E402

with open(os.path.join(ROOT, 'renet_b200', 'csrc', 'common.cuh')) as fh:
    MIN_ROWS = int(re.search(r'kDedupMinRows = (\d+);', fh.read()).group(1))

L = _lib.lib()
dev = 'cuda:0'
PAD = 64          # rows past M that must stay untouched
K = N = 200

torch.manual_seed(0)
_lib.ensure_scratch(dev)
L.renet_set_gemm_engine(1)
L.renet_set_weight_generation(-1)       # no packed-weight cache: every call packs B (one launch)
B = torch.randn(K, N, device=dev) * 0.1
A_ent = torch.randn(23033, K, device=dev) * 0.3


def gemm(A, idx, M):
    out = torch.full((M + PAD, N), float('nan'), device=dev)
    n0 = _lib.launch_count()
    _lib.check(L.renet_selfloop_gemm(_lib.ptr(A), _lib.ptr(idx), _lib.ptr(B), _lib.ptr(out), M, K, N, _lib.stream()),
               'renet_selfloop_gemm')
    return out, _lib.launch_count() - n0


def check(name, A, idx):
    M = idx.numel()
    got, launches = gemm(A, idx, M)
    ref, _ = gemm(A[idx.long()].contiguous(), None, M)
    torch.cuda.synchronize()
    dedup = M >= MIN_ROWS
    # pack + GEMM, or pack + dedupe + GEMM over the distinct rows + expand
    assert launches == (4 if dedup else 2), '%s: %d launches' % (name, launches)
    assert not torch.isnan(got[:M]).any(), '%s: outputs left unwritten' % name
    assert torch.isnan(got[M:]).all(), '%s: rows past M were written' % name
    assert torch.equal(got[:M], ref[:M]), '%s: differs from the plain product, max %.3e' % (
        name, (got[:M] - ref[:M]).abs().max().item())
    print('%-28s M=%6d distinct=%6d dedup=%s ok' % (name, M, torch.unique(idx).numel(), dedup))


def rand_idx(M, rows):
    return torch.randint(0, rows, (M,), device=dev, dtype=torch.int32)


check('random over 23033', A_ent, rand_idx(34500, 23033))
check('one value', A_ent, torch.full((34500,), 4711, device=dev, dtype=torch.int32))
check('all distinct', A_ent, torch.randperm(23033, device=dev)[:20000].int())
hubs = torch.tensor([3, 17, 9000, 15000, 23032], device=dev, dtype=torch.int32)
hub_heavy = torch.where(torch.rand(34500, device=dev) < 0.9, hubs[torch.randint(0, 5, (34500,), device=dev)],
                        rand_idx(34500, 23033))
check('hub-heavy', A_ent, hub_heavy)
check('just below the threshold', A_ent, rand_idx(MIN_ROWS - 1, 23033))
check('at the threshold', A_ent, rand_idx(MIN_ROWS, 23033))

# consecutive calls of one size (one table size): the second call's indices partly repeat the first's in another order, so a
# key left by the first call that were taken for a match would hand out the first call's row numbers
first = torch.randperm(23033, device=dev)[:18000].int()
second = torch.cat((first[9000:], torch.randperm(23033, device=dev)[:9000].int()))[torch.randperm(18000, device=dev)]
check('consecutive call 1', A_ent, first[torch.randint(0, 18000, (30000,), device=dev)])
check('consecutive call 2', A_ent, second[torch.randint(0, 18000, (30000,), device=dev)])

# indices that collide under the table's hash (Fibonacci hashing of the index into 2^bits >= 2M slots): every index whose
# slot falls into one 32-slot band, over an A of 2^20 rows, so they all probe through one cluster
M = 20000
bits = int(np.ceil(np.log2(2 * M)))
v = np.arange(1 << 20, dtype=np.uint64)
slot = ((v * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)) >> np.uint64(32 - bits)
band = v[(slot >= 1000) & (slot < 1032)].astype(np.int64)
same = v[slot == 1000].astype(np.int64)
assert band.size > 300 and same.size >= 8, (band.size, same.size)
A_big = torch.randn(1 << 20, K, device=dev) * 0.3
pool = torch.from_numpy(np.concatenate([band, same, same])).to(dev).int()
check('colliding indices', A_big, pool[torch.randint(0, pool.numel(), (M,), device=dev)])
print('DEDUP_OK')
