"""Build libnar_b200.so (sm_90a only) in-tree with nvcc.  No torch extension machinery:
the product is a plain C-ABI shared library (include/nar_b200.h) loaded with ctypes."""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libnar_b200.so')
SOURCES = ['gemm_wgmma.cu', 'features.cu', 'sampler.cu', 'rnn.cu', 'loss.cu', 'misc.cu', 'host_state.cu', 'state.cu', 'car.cu',
           'gru.cu', 'recommend.cu', 'engine.cu', 'baselines.cu', 'sknn.cu',
           'eval_metrics.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17', '-diag-suppress', '128',
              '-Xcompiler', '-fPIC']


def _nvcc() -> str:
    for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return 'nvcc'


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force: bool = False, verbose: bool = False) -> str:
    hdrs = [os.path.join(CSRC, 'common.cuh'), os.path.join(HERE, '..', 'include', 'nar_b200.h')]
    objdir = os.path.join(HERE, '..', 'build', 'obj')
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace('.cu', '.o'))
        if force or _stale(o, [s] + hdrs):
            jobs.append([nvcc] + NVCC_FLAGS + ['-c', s, '-o', o])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed: %s\n%s\n%s' % (' '.join(cmd), r.stdout, r.stderr))
        if verbose and (r.stdout or r.stderr):
            print(r.stdout, r.stderr, file=sys.stderr)

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    objs = [os.path.join(objdir, s.replace('.cu', '.o')) for s in SOURCES]
    if force or jobs or _stale(LIB, objs):
        run([nvcc, '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a'])
    return LIB


if __name__ == '__main__':
    print(build_library(force='--force' in sys.argv, verbose=True))
