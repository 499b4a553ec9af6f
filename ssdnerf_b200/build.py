"""Builds libssdnerf_b200.so in-tree with nvcc for sm_90a (no JIT cache: the .so travels with the repo).

Every csrc/*.cu is compiled to an object under ssdnerf_b200/_obj/ (git-ignored) in parallel and only when it or a header changed,
then linked; `python -m ssdnerf_b200.build [--force] [-v]`."""
import glob
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(HERE, '_obj')
LIB = os.path.join(HERE, 'libssdnerf_b200.so')

NVCC_FLAGS = [
    '-O3', '-std=c++17', '-lineinfo',
    '-gencode', 'arch=compute_90a,code=sm_90a',
    '-Xcompiler', '-fPIC,-fvisibility=hidden',
    '--expt-relaxed-constexpr',
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')))


def _headers():
    return glob.glob(os.path.join(CSRC, '*.cuh')) + glob.glob(os.path.join(HERE, '..', 'include', '*.h'))


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in sources() + _headers())


def build_lib(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    os.makedirs(OBJ, exist_ok=True)
    hdr_t = max(os.path.getmtime(h) for h in _headers())

    def compile_one(src):
        obj = os.path.join(OBJ, os.path.basename(src)[:-3] + '.o')
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(src), hdr_t):
            return obj, ''
        cmd = [nvcc] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', '-o', obj, src]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if res.returncode != 0:
            sys.stderr.write(res.stdout)
            raise RuntimeError(f'nvcc failed on {src}')
        return obj, res.stdout

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        results = list(ex.map(compile_one, sources()))
    stale = set(glob.glob(os.path.join(OBJ, '*.o'))) - {o for o, _ in results}
    for o in stale:
        os.remove(o)
    res = subprocess.run([nvcc, '-shared', '-cudart', 'shared', '-o', LIB] + [o for o, _ in results] + ['-lcuda'] * 0,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout)
        raise RuntimeError('nvcc failed linking libssdnerf_b200.so')
    if verbose:
        print(''.join(out for _, out in results))
    return LIB


if __name__ == '__main__':
    build_lib(force='--force' in sys.argv, verbose='-v' in sys.argv)
    print(LIB)
