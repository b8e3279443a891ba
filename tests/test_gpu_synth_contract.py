"""-m gpu: the 1M-entity benchmark shard (bench.py --workload synth1m) per row against float64, forward and backward, at the
shape bench.py measures (tests/synth_contract_check.py lists the stages, bars and mistakes).  Each shard runs in a
subprocess under a timeout, as the GEMM and GRU contracts do: the recurrence is one cooperative launch whose grid barrier
traps rather than hangs, so a fault can only fail this test.  The report (err / bar per stage and gradient, the serving
kernels, the mistakes' misses, wall time and peak memory) is written past pytest's capture."""
import gc
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(request, args, timeout):
    # the shard's restatements need tens of GB: hand back what this process's allocator caches from earlier tests
    torch = sys.modules.get('torch')
    if torch is not None and torch.cuda.is_initialized():
        gc.collect()
        torch.cuda.empty_cache()
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'synth_contract_check.py')] + args, capture_output=True,
                       text=True, timeout=timeout)
    with request.config.pluginmanager.getplugin('capturemanager').global_and_fixture_disabled():
        sys.stdout.write('\n' + r.stdout)
        sys.stdout.write(r.stderr[-3000:])
    return r


def test_synth1m_forward_backward(request):
    """the bench's shard: N = 1 000 000 (--synth-nodes' default), every stage of the step and of its backward"""
    r = run(request, ['--nodes', '1000000'], 900)
    assert r.returncode == 0 and 'SYNTH_CONTRACT_OK' in r.stdout


def test_synth4m_forward(request):
    """bench.py --synth-nodes 4194304: the forward stages on a shard of 4 M nodes and 134 M edges"""
    r = run(request, ['--nodes', '4194304', '--forward-only'], 900)
    assert r.returncode == 0 and 'SYNTH_CONTRACT_OK' in r.stdout
