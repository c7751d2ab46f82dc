#!/usr/bin/env python
"""Build libyolo2_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python yolo2-pytorch_b200/build.py [--force] [--verbose]

One object per translation unit (parallel), then a shared library with the static CUDA runtime so
it does not depend on which libcudart the hosting process (PyTorch) loaded.  The .so and the
objects are build products (git-ignored).
"""
import argparse
import concurrent.futures
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT = os.path.join(HERE, 'libyolo2_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17', '-Xcompiler', '-fPIC',
         '--expt-relaxed-constexpr', '-Xptxas', '-v']


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith('.cu'))


def newest_src_mtime():
    return max(os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC))


def compile_one(src, verbose):
    obj = os.path.join(CSRC, src[:-3] + '.o')
    cmd = [NVCC] + FLAGS + ['-c', os.path.join(CSRC, src), '-o', obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (src, r.stdout, r.stderr))
    return obj, r.stderr if verbose else ''


def build(force=False, verbose=False):
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= newest_src_mtime():
        return OUT
    with concurrent.futures.ThreadPoolExecutor(max_workers=8) as ex:
        results = list(ex.map(lambda s: compile_one(s, verbose), sources()))
    objs = [o for o, _ in results]
    if verbose:
        for _, log in results:
            sys.stderr.write(log)
    cmd = [NVCC, '-shared', '-o', OUT] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a', '-Xcompiler', '-fPIC', '-ldl']
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    return OUT


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--force', action='store_true')
    ap.add_argument('--verbose', action='store_true')
    a = ap.parse_args()
    print(build(a.force, a.verbose))
