"""-m gpu: the whole encoder -- batching, renet_prepare_sequences, renet_encode_fwd with its side-stream fork, the fallback
and the training path's backward chain -- per query row and per gradient row against the float64 restatement, each case
first showing in float64 that it can see the simulated mistakes (tests/encoder_contract_check.py lists the paths, the bar,
the mistakes and the cases)."""
import sys

import pytest
import torch

import encoder_contract_check as chk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def report(request):
    """after the module's cases: the largest err / bar per path and output, and the smallest miss per mistake"""
    assert torch.cuda.is_available()
    yield
    with request.config.pluginmanager.getplugin('capturemanager').global_and_fixture_disabled():
        sys.stdout.write('\nencoder contract on %s, tau %g (forward) / %g (gradients):\n  %s\n' % (
            torch.cuda.get_device_name(0), chk.TAU_FWD, chk.TAU_GRAD, '\n  '.join(chk.summary())))


@pytest.mark.parametrize('name', sorted(chk.CASES))
def test_encoder_contract(name):
    before = torch.are_deterministic_algorithms_enabled()
    from renet_b200 import _lib
    engine = _lib.lib().renet_get_gemm_engine()
    chk.CASES[name]()
    assert torch.are_deterministic_algorithms_enabled() == before, 'the case left deterministic mode changed'
    assert _lib.lib().renet_get_gemm_engine() == engine, 'the case left the GEMM engine changed'
