"""The numpy Philox4x32-10 that tests/support_contract_check.py checks the dropout masks against: Random123's published
known answers, and the constants and round structure of the CUDA toolkit's curand_Philox4x32_10 (no GPU needed)."""
import os
import re

import numpy as np
import pytest

import support_contract_check as chk


def words(*w):
    return tuple(np.array([x], dtype=np.uint64) for x in w)


@pytest.mark.parametrize('ctr, key, expect', [
    # Random123 kat_vectors, philox4x32 10 rounds
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, expect):
    got = chk.philox4x32_10(words(*ctr), key)[0]
    assert tuple(int(x) for x in got) == expect, [hex(int(x)) for x in got]


def test_philox_constants_match_curand():
    cuda = os.environ.get('CUDA_HOME', '/usr/local/cuda')
    path = os.path.join(cuda, 'include', 'curand_philox4x32_x.h')
    if not os.path.exists(path):
        pytest.skip('no CUDA toolkit headers')
    src = open(path).read()
    const = {k: int(v, 16) for k, v in re.findall(r'#define (PHILOX_\w+)\s+\((0x[0-9A-Fa-f]+)\)', src)}
    assert (const['PHILOX_M4x32_0'], const['PHILOX_M4x32_1']) == (chk.PHILOX_M0, chk.PHILOX_M1)
    assert (const['PHILOX_W32_0'], const['PHILOX_W32_1']) == (chk.PHILOX_W0, chk.PHILOX_W1)
    body = src[src.index('QUALIFIERS uint4 curand_Philox4x32_10'):]
    body = body[:body.index('}')]
    assert body.count('_philox4x32round(c, k)') == 10          # ten rounds, the key bumped between them
    assert 'ret  = {hi1^ctr.y^key.x, lo1, hi0^ctr.w^key.y, lo0}' in src


def test_mask_layout():
    """word idx & 3 of counter idx >> 2; scale 1/(1-p) in fp32 where (float)w * 2^-32 >= p"""
    seed, off, n, p = (7 << 32) | 3, 2, 9, 0.5
    m = chk.mask_ref(seed, off, n, p)
    for i in range(n):
        idx = off + i
        r = chk.philox4x32_10(words(idx >> 2, 0, 0, 0), (seed & 0xffffffff, seed >> 32))[0]
        u = np.float32(r[idx & 3]) * np.float32(2.0 ** -32)
        assert m[i] == (np.float32(2.0) if u >= np.float32(p) else np.float32(0.0))
    assert chk.mask_ref(seed, 0, 64, 0.0).tolist() == [1.0] * 64


@pytest.mark.parametrize('seed, off, n, p', [(0x1234_5678_9ABC_DEF1, 0, 4099, 0.5), (0x0DDBA11_5EED, 3, 1001, 0.5),
                                             (42, (1 << 34) - 6, 37, 0.5), ((1 << 64) - 1, 5, 517, 0.9), (7, 2, 64, 0.0)])
def test_torch_mask_port(seed, off, n, p):
    """the training-step suite's torch port of mask_ref (run here on the CPU): the same scale factors, counters whose high
    word turns non-zero and an all-ones key included"""
    import torch
    import step_contract_check as step
    got = step.mask_torch(seed, off, n, p, device='cpu')
    assert got.dtype == torch.float32
    np.testing.assert_array_equal(got.numpy(), chk.mask_ref(seed, off, n, p))
