"""-m gpu: the deduplicated indexed self-loop product (each distinct index computed once, rows copied out) is bitwise equal
to the plain product on the materialised rows, for random, repeated, distinct, hub-heavy, threshold-edge, consecutive and
hash-colliding index patterns.  Run in a subprocess under a timeout, like the other wgmma checks."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_selfloop_dedup_bitwise():
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'selfloop_dedup_check.py')], capture_output=True,
                       text=True, timeout=300)
    sys.stdout.write(r.stdout)
    sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0 and 'DEDUP_OK' in r.stdout
