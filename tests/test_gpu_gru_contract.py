"""-m gpu: the fused GRU forward and backward against a float64 reference at the recurrence kernel's schedule edges
(tests/gru_contract_check.py), run in a subprocess under a timeout like the other kernel checks: the recurrence is one
cooperative launch whose grid barrier traps rather than hangs, so a fault can only fail this test."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gru_forward_backward_contract():
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'gru_contract_check.py')], capture_output=True, text=True,
                       timeout=600)
    sys.stdout.write(r.stdout)
    sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0 and 'GRU_CONTRACT_OK' in r.stdout
