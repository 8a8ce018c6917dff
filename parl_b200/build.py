"""Build libparl_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m parl_b200.build [--force] [-v]

One translation unit per .cu under parl_b200/csrc, compiled in parallel, linked
into parl_b200/csrc/libparl_b200.so (static cudart: the library carries no torch
or libcudart.so dependency, so any host — ctypes, cgo, JNI — can load it).
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'csrc')
LIB = os.path.join(CSRC, 'libparl_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
FLAGS = ARCH + ['-lineinfo', '-O3', '-std=c++17',
        '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr']


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith('.cu'))


def _stamp():
    h = hashlib.sha1()
    for f in sorted(os.listdir(CSRC)):
        if f.endswith(('.cu', '.cuh', '.h')):
            h.update(f.encode())
            with open(os.path.join(CSRC, f), 'rb') as fh:
                h.update(fh.read())
    with open(os.path.join(CSRC, '..', '..', 'include', 'parl_b200.h'), 'rb') as fh:
        h.update(fh.read())
    h.update(' '.join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    stamp_file = os.path.join(CSRC, 'build', 'stamp')
    stamp = _stamp()
    if not force and os.path.exists(LIB) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return LIB
    if not os.path.exists(NVCC):
        if os.path.exists(LIB):
            return LIB          # GPU box without a toolkit: use the prebuilt library that travelled
        raise RuntimeError('nvcc not found at %s and no prebuilt %s' % (NVCC, LIB))
    os.makedirs(os.path.join(CSRC, 'build'), exist_ok=True)

    def compile_one(src):
        obj = os.path.join(CSRC, 'build', src[:-3] + '.o')
        cmd = [NVCC] + FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', os.path.join(CSRC, src), '-o', obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (src, r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, _sources()))
    cmd = [NVCC, '-shared'] + ARCH + ['-o', LIB] + objs
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    with open(stamp_file, 'w') as f:
        f.write(stamp)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
