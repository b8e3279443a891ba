"""-m gpu: the training step's support kernels -- clip + Adam, row scatter, segment pooling, the self-loop backward, the
dropout masks and the device graph builders -- per element against float64 or an exact restatement, with the kernels that
served each case asserted from their profiled names (tests/support_contract_check.py lists the references, the bars and
the cases)."""
import sys

import pytest
import torch

import support_contract_check as chk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def report(request):
    """after the module's cases: the largest error / bound per kernel, past pytest's capture"""
    assert torch.cuda.is_available()
    yield
    with request.config.pluginmanager.getplugin('capturemanager').global_and_fixture_disabled():
        sys.stdout.write('\nsupport contract on %s (error / bound, 0 = exact):\n  %s\n' % (torch.cuda.get_device_name(0),
                                                                                         '\n  '.join(chk.summary())))


@pytest.mark.parametrize('name', sorted(chk.CASES))
def test_support_contract(name):
    before = torch.are_deterministic_algorithms_enabled()
    chk.CASES[name]()
    assert torch.are_deterministic_algorithms_enabled() == before, 'the case left deterministic mode changed'
