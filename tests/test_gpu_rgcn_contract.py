"""-m gpu: the RGCN gather kernels (stream and tile), the dH kernels and the dW kernels per row against float64 on every
kernel path, with the kernel that served each case asserted from its profiled name (tests/rgcn_contract_check.py lists
the cases and the branch each one exists for)."""
import sys

import pytest
import torch

import rgcn_contract_check as chk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def report(request):
    """after the module's cases: the largest error ratio per kernel, past pytest's capture"""
    assert torch.cuda.is_available()
    yield
    with request.config.pluginmanager.getplugin('capturemanager').global_and_fixture_disabled():
        sys.stdout.write('\nrgcn contract on %s, bar C = %g:\n  %s\n' % (torch.cuda.get_device_name(0), chk.C,
                                                                        '\n  '.join(chk.summary())))


@pytest.mark.parametrize('name', sorted(chk.CASES))
def test_rgcn_contract(name):
    chk.CASES[name]()
