"""-m "not gpu": librenet_b200.so builds for sm_90a, loads, and exports every symbol include/renet_b200.h
declares (no compute calls here: these tests run without a GPU)."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def so_path():
    from renet_b200 import build
    return build.build()


def _declared():
    txt = open(os.path.join(ROOT, 'include', 'renet_b200.h')).read()
    txt = re.sub(r'/\*.*?\*/', '', txt, flags=re.S)
    return sorted(set(re.findall(r'\b(renet_[a-z0-9_]+)\s*\(', txt)))


def test_header_symbols_exported(so_path):
    names = _declared()
    assert len(names) >= 12
    lib = ctypes.CDLL(so_path)
    for n in names:
        assert hasattr(lib, n), 'missing export: ' + n


def test_python_binding_covers_header(so_path):
    from renet_b200 import _lib
    assert sorted(_lib.SIGNATURES) == _declared()
    L = _lib.lib()
    assert L.renet_version() >= 100
    assert L.renet_last_error() == b''
    assert L.renet_csr_workspace_bytes(1000, 5000) > 0          # host-only size query
    assert L.renet_gru_workspace_bytes(100, 10, 5, 200) > 0


def test_argument_validation_needs_no_gpu(so_path):
    from renet_b200 import _lib
    L = _lib.lib()
    rc = L.renet_rgcn_block_fwd(None, None, None, None, None, None, None, None, None, 10, 5, 200, 200, 7, 4, 1, None)
    assert rc == -1 and b'num_bases' in L.renet_last_error()
    rc = L.renet_rgcn_block_fwd(None, None, None, None, None, None, None, None, None, 10, 5, 200, 200, 100, 4, 1, None)
    assert rc == -1 and b'null pointer' in L.renet_last_error()
    # renet_debug_gemm rejects null operands and kernels forced where their preconditions do not hold, before any launch
    # (the fake addresses below are never dereferenced)
    fake = [ctypes.c_void_p(4096 * (i + 1)) for i in range(4)]
    ws = ctypes.c_void_p(1 << 20)

    def gemm(form, kernel, K=200, A=fake[0], idx=None, C=fake[2], acc=0, batch=1, ws_bytes=1 << 30):
        return L.renet_debug_gemm(form, kernel, A, idx, K, fake[1], 200, C, 200, None, 1000, 200, K, acc, batch, 0, 0, 0, ws,
                                  ws_bytes, None)
    for args, msg in (
            (dict(form=0, kernel=0, A=None), b'null pointer'),
            (dict(form=1, kernel=0, C=None), b'null pointer'),
            (dict(form=3, kernel=0), b'unknown form'),
            (dict(form=0, kernel=7), b'unknown kernel'),
            (dict(form=0, kernel=5, K=228), b'resident kernel needs K <= 224'),    # RESIDENT past its panel size
            (dict(form=1, kernel=6, idx=fake[3]), b'cannot serve'),              # DEDUP outside the nn form
            (dict(form=0, kernel=6, idx=fake[3], acc=1), b'no accumulate'),       # DEDUP accumulating
            (dict(form=0, kernel=3), b'unknown kernel'),                         # 3: the retired kernel id
            (dict(form=0, kernel=1, A=ctypes.c_void_p(4100)), b'tiled FFMA'),     # FFMA_TILED on an unaligned operand
            (dict(form=2, kernel=5), b'FFMA kernels only'),                       # the tn form on a tensor-core kernel
            (dict(form=0, kernel=4, A=ctypes.c_void_p(4100)), b'16-byte aligned'),  # STREAMING on an unaligned operand
            (dict(form=1, kernel=0, ws_bytes=1000), b'workspace'),                # too small a workspace for the packed B
            (dict(form=0, kernel=0, batch=2), b'bad shape')):                     # batches only in the prepacked form
        assert gemm(**args) == -1, args
        assert msg in L.renet_last_error(), (args, L.renet_last_error())


def test_sass_is_sm90a(so_path):
    from renet_b200 import build
    out = subprocess.run([build.CUOBJDUMP, '-lelf', so_path], capture_output=True, text=True).stdout
    assert 'sm_90a' in out, out


def test_hot_path_never_imports_oracle():
    pkg = os.path.join(ROOT, 'renet_b200')
    for f in os.listdir(pkg):
        if f.endswith('.py'):
            src = open(os.path.join(pkg, f)).read()
            assert not re.search(r'^\s*(from|import)\s+oracle', src, flags=re.M), f


def test_missing_library_fails_loudly(tmp_path, monkeypatch):
    from renet_b200 import _lib
    monkeypatch.setattr(_lib, '_lib', None)
    monkeypatch.setattr(_lib, 'LIB_PATH', str(tmp_path / 'nope.so'))
    with pytest.raises(RuntimeError, match='no CPU or PyTorch fallback'):
        _lib.lib()
