"""-m "not gpu": the kernels of the deterministic mode (renet_set_deterministic) contain no float atomic or reduction, read
from the SASS of the built library.  The same pattern must match the atomic kernels they replace, so the check is known to
be able to fail."""
import re
import subprocess

import pytest

# Every kernel the deterministic mode launches in place of, or next to, an atomic one: patterns on the names cu++filt prints
# (template arguments as (bool)0 / (bool)1; the last one of the templated kernels is DET).  The
# float atomics the mode avoids are listed with their replacements in DESIGN §4.
DETERMINISTIC_KERNELS = [
    r'rgcn_dh_tile_kernel<\(bool\)[01], \(bool\)1>',
    r'rgcn_dw_d200_kernel<\(bool\)[01], \(bool\)1>',
    r'rgcn_dw_reduce_kernel\(',
    r'sgemm_tn_splitk_kernel<\(bool\)[01], \(bool\)1>',
    r'sum_partials_kernel\(',
    r'scatter_keys_kernel\(',
    r'scatter_add_rows_sorted_kernel\(',
    r'dropout_grad_rows_kernel\(',
    r'colsum_accum_kernel<\(bool\)1>',
]
# the atomic kernels of the default mode (positive controls)
ATOMIC_KERNELS = [
    r'rgcn_dw_d200_kernel<\(bool\)[01], \(bool\)0>',
    r'scatter_add_rows_kernel\(',
    r'rgcn_dh_tile_kernel<\(bool\)[01], \(bool\)0>',
    r'sgemm_tn_splitk_kernel<\(bool\)[01], \(bool\)0>',
    r'colsum_accum_kernel<\(bool\)0>',
    r'unpack_inputs_dropout_kernel\(',
]
# a float RED / ATOM in global or shared memory, or the compare-and-swap loop of a shared-memory float atomic
FLOAT_ATOMIC = re.compile(r'\b(RED|REDG|ATOM|ATOMG|ATOMS)\.[A-Z0-9_.]*\bF(16|32|64)|ATOMS\.CAST\.SPIN|\b(ATOM|ATOMG|ATOMS)\.[A-Z0-9_.]*CAS')


@pytest.fixture(scope='module')
def sass():
    """{demangled kernel name: SASS text} of librenet_b200.so"""
    from renet_b200 import build
    so = build.build()
    out = subprocess.run([build.CUOBJDUMP, '-sass', so], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for chunk in re.split(r'\n\s*Function : ', out)[1:]:
        name, _, body = chunk.partition('\n')
        funcs[name.strip()] = body
    filt = build.CUOBJDUMP.replace('cuobjdump', 'cu++filt')
    names = list(funcs)
    demangled = subprocess.run([filt], input='\n'.join(names), capture_output=True, text=True, check=True).stdout.split('\n')
    return {d: funcs[n] for n, d in zip(names, demangled)}


def _matching(sass, pattern):
    found = {n: body for n, body in sass.items() if re.search(pattern, n)}
    assert found, 'no kernel matches %r' % pattern
    return found


@pytest.mark.parametrize('pattern', DETERMINISTIC_KERNELS)
def test_deterministic_kernels_have_no_float_atomics(sass, pattern):
    for name, body in _matching(sass, pattern).items():
        hits = [ln.strip() for ln in body.split('\n') if FLOAT_ATOMIC.search(ln)]
        assert not hits, '%s: %s' % (name, hits[:3])


@pytest.mark.parametrize('pattern', ATOMIC_KERNELS)
def test_the_pattern_finds_the_atomic_kernels(sass, pattern):
    for name, body in _matching(sass, pattern).items():
        assert FLOAT_ATOMIC.search(body), name
