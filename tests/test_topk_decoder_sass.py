"""-m "not gpu": the SASS of the per-row top-k with exclusion lists (renet_decoder_topk), read from the built library.

* Its kernels (the EXCL instantiations of the tau and final kernels) hold no float RED / ATOM: the output is reproducible.
* The kernels renet_decoder_group_topk launches -- the (bool)0 instantiations of the same two kernel templates, the EPI 1
  and EPI 5 passes of the packed GEMM and ce_reduce_kernel -- are instruction for instruction what they were before the
  EXCL instantiations were added: tests/golden/group_topk_sass.json holds the digests of their instruction text from that
  build, with the nvcc release that made it (another release compiles differently, and the comparison is skipped)."""
import hashlib
import json
import os
import re
import subprocess

import pytest

from test_deterministic_sass import FLOAT_ATOMIC, _matching, sass  # noqa: F401  (sass is a fixture)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'group_topk_sass.json')
# the group top-k's kernels, by the names cu++filt prints; the key is the name without the template argument it gained
GROUP_TOPK = {
    'topk_tau_kernel': r'topk_tau_kernel<\(bool\)0>',
    'topk_final_kernel': r'topk_final_kernel<\(bool\)0>',
    'umma_gemm_packed_kernel<0,1>': r'umma_gemm_packed_kernel<\(bool\)0, \(int\)1>',
    'umma_gemm_packed_kernel<0,5>': r'umma_gemm_packed_kernel<\(bool\)0, \(int\)5>',
    'ce_reduce_kernel': r'::ce_reduce_kernel\(',
}


def instruction_digest(body):
    """sha256 of a function's instructions, one per line, without their addresses and encodings."""
    lines = [re.sub(r'/\*[0-9a-f]{4}\*/', '', ln).split(';')[0].strip() for ln in body.split('\n')
             if re.search(r'/\*[0-9a-f]{4}\*/', ln)]
    return hashlib.sha256('\n'.join(lines).encode()).hexdigest()


def _nvcc_release():
    from renet_b200 import build
    out = subprocess.run([build.NVCC, '--version'], capture_output=True, text=True, check=True).stdout
    return re.search(r'release [0-9.]+, V[0-9.]+', out).group(0)


@pytest.mark.parametrize('kernel', ['topk_tau_kernel', 'topk_final_kernel'])
def test_exclusion_kernels_have_no_float_atomics(sass, kernel):  # noqa: F811
    found = _matching(sass, kernel + r'<\(bool\)1>')
    assert len(found) == 1, sorted(found)
    for name, body in found.items():
        hits = [ln.strip() for ln in body.split('\n') if FLOAT_ATOMIC.search(ln)]
        assert not hits, '%s: %s' % (name, hits[:3])


@pytest.mark.parametrize('kernel', list(GROUP_TOPK))
def test_group_topk_kernels_unchanged(sass, kernel):  # noqa: F811
    golden = json.load(open(GOLDEN))
    if _nvcc_release() != golden['nvcc']:
        pytest.skip('the digests were recorded with nvcc %s' % golden['nvcc'])
    found = _matching(sass, GROUP_TOPK[kernel])
    assert len(found) == 1, sorted(found)
    assert instruction_digest(next(iter(found.values()))) == golden['kernels'][kernel], kernel
