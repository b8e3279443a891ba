"""-m "not gpu": renet_decoder_topk rejects bad arguments on the host, before any launch, as its sibling decoder entries do:
its shape and k, its capacity, exclusion lists without ranges, null pointers, the workspace size and the 16-byte alignment
of X and W; and it returns at once when there are no rows.  The header, the .so and the binding agree on it.

Cases that pass made-up device addresses run only where there is no CUDA device (see test_decoder_args.py)."""
import ctypes
import threading

import pytest
import torch

ARGS = 'X W bias excl_col excl_begin excl_end M N K k capacity values indices needed ws ws_bytes stream'.split()
SCALARS = dict(M=64, N=1000, K=200, k=10, capacity=1000)
REQUIRED = 'X W values indices needed ws'.split()

no_fake_addresses_on_a_gpu = pytest.mark.skipif(
    torch.cuda.is_available(), reason='passes made-up device addresses: only where no kernel could be launched on them')


@pytest.fixture(scope='module')
def L():
    from renet_b200 import _lib, build
    build.build()
    return _lib.lib()


def _ws(L, v):
    return int(L.renet_decoder_topk_workspace_bytes(v['M'], v['N'], v['K'], v['capacity']))


def _call(L, fake=True, **over):
    """renet_decoder_topk with distinct made-up addresses (NULL when fake is False; no lists unless given), SCALARS and the
    overrides; (status, error message), on a thread of its own so the last error stays there."""
    v = dict(SCALARS)
    v.update((k, over[k]) for k in over if k in SCALARS)
    args = []
    for i, a in enumerate(ARGS):
        if a == 'ws_bytes':
            args.append(over.get(a, _ws(L, v)))
        elif a in over and a not in SCALARS:
            val = over[a]
            args.append(ctypes.c_void_p(val) if isinstance(val, int) else val)
        elif a in v:
            args.append(v[a])
        elif a == 'stream' or a.startswith('excl_') or a == 'bias':
            args.append(None)
        else:
            args.append(ctypes.c_void_p((i + 1) << 20) if fake else None)
    out = []
    t = threading.Thread(target=lambda: out.append((L.renet_decoder_topk(*args), L.renet_last_error())))
    t.start()
    t.join()
    return out[0]


def test_binding_matches_header(L):
    from renet_b200 import _lib
    assert 'renet_decoder_topk' in _lib.SIGNATURES and 'renet_decoder_topk_workspace_bytes' in _lib.SIGNATURES
    assert len(_lib.SIGNATURES['renet_decoder_topk'][1]) == len(ARGS)
    assert _ws(L, SCALARS) > _ws(L, dict(SCALARS, M=1)) > 0


@pytest.mark.parametrize('over,msg', [
    (dict(K=202), b'multiple of 4'),
    (dict(N=0), b'bad shape'),
    (dict(M=-1), b'bad shape'),
    (dict(k=0), b'outside [1, N'),
    (dict(k=1001), b'outside [1, N'),
    (dict(N=20000, k=16385, capacity=20000), b'RENET_TOPK_MAX_K'),
    (dict(capacity=9), b'capacity 9 < k'),
])
def test_bad_shape_or_k_rejected(L, over, msg):
    rc, err = _call(L, fake=False, **over)
    assert rc == -1 and err.startswith(b'renet_decoder_topk: ') and msg in err, err


@pytest.mark.parametrize('missing', ['excl_begin', 'excl_end', 'both'])
def test_lists_without_ranges_rejected(L, missing):
    over = dict(excl_col=1 << 28, excl_begin=2 << 28, excl_end=3 << 28)
    for a in (['excl_begin', 'excl_end'] if missing == 'both' else [missing]):
        over[a] = None
    rc, err = _call(L, fake=False, **over)
    assert rc == -1 and b'exclusion lists need excl_begin and excl_end' in err, err


def test_zero_rows_return_before_reading_a_pointer(L):
    needed = ctypes.c_int32(-7)
    rc, err = _call(L, fake=False, M=0, needed=ctypes.cast(ctypes.byref(needed), ctypes.c_void_p))
    assert rc == 0, err
    assert needed.value == -7


def test_null_needed_rejected_without_rows(L):
    rc, err = _call(L, fake=False, M=0)
    assert rc == -1 and err == b'renet_decoder_topk: null pointer', err


@no_fake_addresses_on_a_gpu
@pytest.mark.parametrize('pointer', REQUIRED)
def test_null_pointer_rejected(L, pointer):
    rc, err = _call(L, **{pointer: None})
    assert rc == -1 and err == b'renet_decoder_topk: null pointer', err


@no_fake_addresses_on_a_gpu
def test_workspace_one_byte_short_rejected(L):
    rc, err = _call(L, ws_bytes=_ws(L, SCALARS) - 1)
    assert rc == -1 and err == b'renet_decoder_topk: workspace too small', err


@no_fake_addresses_on_a_gpu
@pytest.mark.parametrize('operand', ['X', 'W'])
def test_misaligned_operand_rejected(L, operand):
    rc, err = _call(L, **{operand: (1 << 24) + 4})
    assert rc == -1 and err == b'renet_decoder_topk: X and W must be 16-byte aligned', err
