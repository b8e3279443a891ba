"""-m gpu: every kernel of the dense-GEMM engine in every argument form its callers use, against fp64, with sentinels around
the written window and the serving kernel pinned per case (tests/gemm_contract_check.py).  Run in a subprocess under a
timeout so that a wrong descriptor can only fail this test (the kernels trap instead of hanging), never poison the others."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gemm_engine_contract_matrix():
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'gemm_contract_check.py')], capture_output=True, text=True,
                       timeout=600)
    sys.stdout.write(r.stdout)
    sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0 and 'GEMM_CONTRACT_OK' in r.stdout
