"""-m "not gpu": the decoder's C entries reject bad arguments on the host, before any launch.

renet_decoder_ce_fwd/_bwd, renet_decoder_soft_ce_fwd/_bwd, renet_decoder_group_topk, renet_decoder_rank and
renet_decoder_rank_multi each check their shape, their pointers, their workspace size and the 16-byte alignment of X and W
(the logits GEMM reads both with float4 loads), and return at once when there are no rows.

Most cases pass made-up device addresses: they are never dereferenced when the check holds, but a missing check would
launch kernels on them.  Those tests run only where there is no CUDA device; the cases that pass no made-up address
(a bad shape, no rows) run everywhere."""
import ctypes
import threading

import pytest
import torch

ENTRIES = {   # entry -> its arguments in order; scalars by name, every other name is a pointer
    'renet_decoder_ce_fwd': 'X W bias target loss_rows lse M N K ws ws_bytes stream',
    'renet_decoder_ce_bwd': 'X W bias target lse scale d_scale dX dW dbias M N K ws ws_bytes stream',
    'renet_decoder_soft_ce_fwd': 'X W bias P ldp loss_rows lse psum M N K ws ws_bytes stream',
    'renet_decoder_soft_ce_bwd': 'X W bias P ldp lse psum scale d_scale dX dW dbias M N K ws ws_bytes stream',
    'renet_decoder_group_topk': 'X W bias row_weight G R N K k order capacity values indices needed ws ws_bytes stream',
    'renet_decoder_rank': 'X W bias label excl_col excl_begin excl_end loss_rows counts M N K ws ws_bytes stream',
    'renet_decoder_rank_multi': 'X W bias label n_lists excl_col excl_begin excl_end loss_rows counts M N K ws ws_bytes stream',
}
REQUIRED = {  # the pointers each entry must not be given as NULL
    'renet_decoder_ce_fwd': 'X W target loss_rows lse ws',
    'renet_decoder_ce_bwd': 'X W target lse dX dW ws',
    'renet_decoder_soft_ce_fwd': 'X W P loss_rows lse psum ws',
    'renet_decoder_soft_ce_bwd': 'X W P lse psum dX dW ws',
    'renet_decoder_group_topk': 'X W row_weight values indices needed ws',
    'renet_decoder_rank': 'X W label loss_rows counts ws',
    'renet_decoder_rank_multi': 'X W label loss_rows counts ws',
}
SCALARS = dict(M=64, N=1000, K=200, ldp=1000, scale=1.0, G=4, R=16, k=10, order=0, capacity=1000, n_lists=0)
SOFT = ('renet_decoder_soft_ce_fwd', 'renet_decoder_soft_ce_bwd')

no_fake_addresses_on_a_gpu = pytest.mark.skipif(
    torch.cuda.is_available(), reason='passes made-up device addresses: only where no kernel could be launched on them')


@pytest.fixture(scope='module')
def L():
    from renet_b200 import _lib, build
    build.build()
    return _lib.lib()


def _workspace_bytes(L, name, v):
    if name == 'renet_decoder_group_topk':
        return int(L.renet_decoder_group_topk_workspace_bytes(v['G'], v['R'], v['N'], v['K'], v['capacity']))
    query = {'renet_decoder_ce_fwd': L.renet_decoder_ce_workspace_bytes,
             'renet_decoder_ce_bwd': L.renet_decoder_ce_bwd_workspace_bytes,
             'renet_decoder_soft_ce_fwd': L.renet_decoder_soft_ce_workspace_bytes,
             'renet_decoder_soft_ce_bwd': L.renet_decoder_soft_ce_bwd_workspace_bytes}.get(name, L.renet_decoder_rank_workspace_bytes)
    return int(query(v['M'], v['N'], v['K']))


def _call(L, name, fake=True, **over):
    """Call `name` with distinct 1 MiB-aligned made-up addresses for its pointers (NULL when fake is False), SCALARS for its
    scalars, exactly the workspace it asks for, and the overrides `over` (an int for a pointer is an address).  Returns
    (status, error message).  The call runs on a thread of its own: the library's last error is per thread, so the
    errors provoked here never reach the other tests of the session."""
    v = dict(SCALARS)
    v.update((k, over[k]) for k in over if k in SCALARS)
    args = []
    for i, a in enumerate(ENTRIES[name].split()):
        if a == 'ws_bytes':
            args.append(over.get(a, _workspace_bytes(L, name, v)))
        elif a in over and a not in SCALARS:
            val = over[a]
            args.append(ctypes.c_void_p(val) if isinstance(val, int) else val)
        elif a in v:
            args.append(v[a])
        elif a == 'stream':
            args.append(None)
        else:
            args.append(ctypes.c_void_p((i + 1) << 20) if fake else None)
    out = []
    t = threading.Thread(target=lambda: out.append((getattr(L, name)(*args), L.renet_last_error())))
    t.start()
    t.join()
    return out[0]


@no_fake_addresses_on_a_gpu
@pytest.mark.parametrize('operand', ['X', 'W'])
@pytest.mark.parametrize('name', list(ENTRIES))
def test_misaligned_operand_rejected(L, name, operand):
    """X and W are read with float4 loads: an operand 4 bytes off a 16-byte boundary is refused, by every entry."""
    rc, msg = _call(L, name, **{operand: (1 << 24) + 4})
    assert rc == -1 and msg == name.encode() + b': X and W must be 16-byte aligned', msg


@pytest.mark.parametrize('name', list(ENTRIES))
def test_k_not_multiple_of_4_rejected(L, name):
    rc, msg = _call(L, name, fake=False, K=202)
    assert rc == -1 and name.encode() + b': bad shape' in msg and b'multiple of 4' in msg, msg


@pytest.mark.parametrize('name', SOFT)
def test_soft_target_stride_below_n_rejected(L, name):
    rc, msg = _call(L, name, fake=False, ldp=SCALARS['N'] - 1)
    assert rc == -1 and b'ldp >= N' in msg, msg


@no_fake_addresses_on_a_gpu
@pytest.mark.parametrize('name', list(ENTRIES))
def test_workspace_one_byte_short_rejected(L, name):
    rc, msg = _call(L, name, ws_bytes=_workspace_bytes(L, name, SCALARS) - 1)
    assert rc == -1 and msg == name.encode() + b': workspace too small', msg


@no_fake_addresses_on_a_gpu
@pytest.mark.parametrize('name,pointer', [(n, p) for n in ENTRIES for p in REQUIRED[n].split()])
def test_null_pointer_rejected(L, name, pointer):
    rc, msg = _call(L, name, **{pointer: None})
    assert rc == -1 and msg == name.encode() + b': null pointer', msg


@pytest.mark.parametrize('name', list(ENTRIES))
def test_zero_rows_return_before_reading_a_pointer(L, name):
    """M = 0 (G = 0 groups) returns success with every pointer NULL; the top-k's `needed` flag is checked first, so it gets
    a real host address that is never written."""
    needed = ctypes.c_int32(-7)
    rc, msg = _call(L, name, fake=False, M=0, G=0, needed=ctypes.cast(ctypes.byref(needed), ctypes.c_void_p))
    assert rc == 0, msg
    assert needed.value == -7
