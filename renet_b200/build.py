"""Build librenet_b200.so in-tree with nvcc for sm_90a (H100) only.

    python -m renet_b200.build [--force] [--verbose]

The .so and the object files under csrc/build/ are build products (git-ignored).
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT = os.path.join(HERE, 'librenet_b200.so')
BUILD_DIR = os.path.join(HERE, 'csrc', 'build')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), 'cuobjdump')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
         '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr']


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cu', '.cpp')))


def _digest():
    h = hashlib.sha256()
    files = sources() + sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h')))
    files.append(os.path.join(HERE, '..', 'include', 'renet_b200.h'))
    for f in files:
        with open(f, 'rb') as fh:
            h.update(f.encode() + b'\0' + fh.read())
    h.update(' '.join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(BUILD_DIR, exist_ok=True)
    stamp = os.path.join(BUILD_DIR, 'stamp')
    dig = _digest()
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == dig:
        return OUT
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(BUILD_DIR, os.path.splitext(os.path.basename(src))[0] + '.o')
        cmd = [NVCC] + FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', src, '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            failed = True
            sys.stderr.write('nvcc failed on %s\n' % src)
    if failed:
        raise RuntimeError('librenet_b200.so: compilation failed')
    cmd = [NVCC, '-shared', '-o', OUT] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a']
    subprocess.check_call(cmd)
    with open(stamp, 'w') as fh:
        fh.write(dig)
    return OUT


if __name__ == '__main__':
    path = build(force='--force' in sys.argv, verbose='--verbose' in sys.argv)
    print(path)
