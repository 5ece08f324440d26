"""In-tree nvcc build of libsimclr_b200.so (sm_90a only: H100).

`python -m simclr_b200.build` or `__graft_entry__.build()`.  Objects go to
`simclr_b200/csrc/_build/`, the shared library to `simclr_b200/libsimclr_b200.so`
(both git-ignored; a checkout builds them once).
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT = os.path.join(HERE, 'libsimclr_b200.so')
BUILD = os.path.join(CSRC, '_build')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')

ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
FLAGS = ARCH + ['-lineinfo', '-O3', '-std=c++17',
         '-Xcompiler', '-fPIC,-fvisibility=hidden', '--expt-relaxed-constexpr',
         '-Xptxas', '-v' if os.environ.get('SIMCLR_PTXAS_V') else '-O3']


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith('.cu'))


def _stamp(path):
    h = hashlib.sha1()
    for f in sorted(os.listdir(CSRC)):
        if f.endswith(('.cu', '.cuh', '.h')):
            with open(os.path.join(CSRC, f), 'rb') as fh:
                h.update(fh.read())
    with open(os.path.join(HERE, '..', 'include', 'simclr_b200.h'), 'rb') as fh:
        h.update(fh.read())
    h.update(' '.join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    stamp_file = os.path.join(BUILD, 'stamp')
    stamp = _stamp(CSRC)
    if not force and os.path.exists(OUT) and os.path.exists(stamp_file) and \
            open(stamp_file).read() == stamp:
        return OUT
    if not os.path.exists(NVCC):
        raise RuntimeError('nvcc not found at %s; cannot build %s' % (NVCC, OUT))
    objs = []

    def compile_one(src):
        obj = os.path.join(BUILD, src[:-3] + '.o')
        cmd = [NVCC] + FLAGS + ['-c', os.path.join(CSRC, src), '-o', obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode != 0:
            sys.stderr.write(' '.join(cmd) + '\n' + r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed on %s' % src)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, _sources()))
    cmd = [NVCC, '-shared', '-o', OUT] + objs + ARCH + ['-Xcompiler', '-fPIC']
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError('link failed')
    with open(stamp_file, 'w') as f:
        f.write(stamp)
    return OUT


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
