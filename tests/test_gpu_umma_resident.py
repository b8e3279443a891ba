"""-m gpu: the resident-panel wgmma GEMM (B panel held in shared memory, A fed to wgmma from registers) at the edges of its
tile schedule, run in a subprocess under a timeout so that a wrong descriptor can only fail this test (the kernel traps
instead of hanging).  Its batched, bias and accumulate forms are exercised through the GRU projections
(tests/test_gpu_gru_renet.py)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_resident_gemm_schedule_edges():
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'umma_resident_check.py')], capture_output=True,
                       text=True, timeout=300)
    sys.stdout.write(r.stdout)
    sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0 and 'RESIDENT_OK' in r.stdout
