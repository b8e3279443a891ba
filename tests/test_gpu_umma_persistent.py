"""-m gpu: the persistent, warp-specialised wgmma GEMM at the edges of its work-unit schedule, run in a subprocess under
a timeout so that a wrong descriptor can only fail this test (the kernel traps instead of hanging)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_persistent_gemm_schedule_edges_and_fused_epilogues():
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'umma_persistent_check.py')], capture_output=True,
                       text=True, timeout=300)
    sys.stdout.write(r.stdout)
    sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0 and 'PERSISTENT_OK' in r.stdout
