"""-m "not gpu": the programmatic-dependent-launch kernels (DESIGN §4), read from the SASS of the built library.

* Trigger after wait: in every kernel the library launches with PDL, each PREEXIT (griddepcontrol.launch_dependents)
  comes after an ACQBULK (griddepcontrol.wait) in the instruction stream, and the backward stream gather does not trigger.
* The stream gather's and the resident GEMM's register, stack and shared-memory figures are those of the build before
  the PDL changes (cuobjdump -res-usage), so the prologue split costs no occupancy and adds no spill."""
import re
import subprocess

import pytest

from test_deterministic_sass import _matching, sass  # noqa: F401  (sass is a fixture)

PDL_KERNELS = [
    r'rgcn_gather_stream_kernel<\(bool\)[01], \(bool\)[01], \(bool\)[01], \(bool\)0,',
    r'umma_gemm_resident_kernel<\(bool\)[01]>',
    r'::dedup_insert_kernel\(',
    r'::dedup_expand_kernel\(',
    r'::umma_pack_b_kernel\(',
]
# (REG, STACK) per kernel, mangled-name pattern -> figures; every one has the static shared memory SHARED:1024
RESOURCES = {
    r'rgcn_gather_stream_kernelILb1ELb1ELb1ELb0ENS_5StCfgILi32ELi2ELi49ELb0ELi64E': (64, 0),   # layer 1, hubs
    r'rgcn_gather_stream_kernelILb1ELb1ELb1ELb0ENS_5StCfgILi32ELi2ELi82ELb0ELi0E': (64, 0),
    r'rgcn_gather_stream_kernelILb0ELb1ELb0ELb0ENS_5StCfgILi32ELi2ELi82ELb0ELi0E': (64, 0),   # read-out sub-graph
    r'umma_gemm_resident_kernelILb0E': (168, 0),
    r'umma_gemm_resident_kernelILb1E': (168, 8),
}


def _ops(body):
    return [m.group(1) for m in re.finditer(r'/\*[0-9a-f]{4}\*/\s+(ACQBULK|PREEXIT)\b', body)]


@pytest.mark.parametrize('pattern', PDL_KERNELS)
def test_trigger_comes_after_wait(sass, pattern):
    for name, body in _matching(sass, pattern).items():
        ops = _ops(body)
        assert 'ACQBULK' in ops and 'PREEXIT' in ops, (name, ops)
        assert ops.index('PREEXIT') > ops.index('ACQBULK'), (name, ops)


def test_backward_stream_gather_does_not_trigger(sass):
    for name, body in _matching(sass, r'rgcn_gather_stream_kernel<.*\(bool\)1, renet::StCfg').items():
        assert 'PREEXIT' not in _ops(body), name


def test_resource_figures_unchanged():
    from renet_b200 import build
    so = build.build()
    out = subprocess.run([build.CUOBJDUMP, '-res-usage', so], capture_output=True, text=True, check=True).stdout
    usage = dict(re.findall(r'Function (\S+):\n\s+(REG:\d+ STACK:\d+ SHARED:\d+ LOCAL:\d+)', out))
    for pattern, (reg, stack) in RESOURCES.items():
        found = {n: u for n, u in usage.items() if re.search(pattern, n)}
        assert found, pattern
        for n, u in found.items():
            assert u == 'REG:%d STACK:%d SHARED:1024 LOCAL:0' % (reg, stack), (n, u)
