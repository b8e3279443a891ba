"""-m gpu: the whole global model -- the pre-training step's s_q rows, targets, loss and gradient rows, the global-embedding
table across its chunks, and predict -- per row against the float64 restatement at the synthetic ICEWS18 and GDELT shapes,
each case first showing in float64 that it can see the simulated mistakes (tests/global_contract_check.py lists the bar,
the mistakes and the cases)."""
import sys
import time

import pytest
import torch

import global_contract_check as chk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def report(request):
    """after the module's cases: the largest err / bar per output, the smallest miss per mistake, the near-tie columns and
    the wall time"""
    assert torch.cuda.is_available()
    t0 = time.perf_counter()
    yield
    with request.config.pluginmanager.getplugin('capturemanager').global_and_fixture_disabled():
        sys.stdout.write('\nglobal-model contract on %s, tau %g (rows) / %g (gradients), %.0f s:\n  %s\n' % (
            torch.cuda.get_device_name(0), chk.TAU_FWD, chk.TAU_GRAD, time.perf_counter() - t0, '\n  '.join(chk.summary())))


@pytest.mark.parametrize('name', sorted(chk.CASES))
def test_global_contract(name):
    before = torch.are_deterministic_algorithms_enabled()
    chk.CASES[name]()
    assert torch.are_deterministic_algorithms_enabled() == before, 'the case left deterministic mode changed'
