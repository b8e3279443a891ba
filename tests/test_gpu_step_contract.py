"""-m gpu: the RE-Net training step -- DataParallelTrainer.train_step with dropout, both directions, backward and the native
clip + Adam over the flat buffers -- per row against float64 at the datasets' shapes over several steps, each case first
showing in float64 that it can see the simulated mistakes (tests/step_contract_check.py lists the bars, the mistakes and
the cases)."""
import sys
import time

import pytest
import torch

import step_contract_check as chk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def report(request):
    """after the module's cases: the largest err / bar per output, the smallest miss per mistake and the wall time"""
    assert torch.cuda.is_available()
    t0 = time.perf_counter()
    yield
    with request.config.pluginmanager.getplugin('capturemanager').global_and_fixture_disabled():
        sys.stdout.write('\ntraining-step contract on %s, tau %g (rows) / %g (gradients), %.0f s:\n  %s\n' % (
            torch.cuda.get_device_name(0), chk.TAU_FWD, chk.TAU_GRAD, time.perf_counter() - t0, '\n  '.join(chk.summary())))


@pytest.mark.parametrize('name', sorted(chk.CASES))
def test_step_contract(name):
    before = torch.are_deterministic_algorithms_enabled()
    from renet_b200 import _lib
    engine = _lib.lib().renet_get_gemm_engine()
    chk.CASES[name]()
    assert torch.are_deterministic_algorithms_enabled() == before, 'the case left deterministic mode changed'
    assert _lib.lib().renet_get_gemm_engine() == engine, 'the case left the GEMM engine changed'
