"""Builds libcapb200.so (the C-ABI shared library, include/capb200.h) in-tree with nvcc for sm_90a (H100).

    python imagecaptioning.pytorch_b200/build.py [--force]

nvcc cross-compiles without a GPU; the resulting .so and the object files are build products (git-ignored).
"""
from __future__ import annotations

import concurrent.futures
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, 'csrc')
OBJ = os.path.join(PKG, 'build')
LIB = os.path.join(PKG, 'libcapb200.so')
SOURCES = ['gemm_tc.cu', 'gemm_simt.cu', 'pointwise.cu', 'vocab.cu', 'beam.cu', 'reward.cu', 'diversity.cu', 'coco_eval.cu', 'transformer.cu', 'attn_tiled.cu', 'gemm_generic.cu', 'gemm_tf32.cu', 'scst_kernels.cu', 'aoa_train_kernels.cu', 'tfm_train_kernels.cu', 'optim.cu', 'engine.cu', 'tfm_engine.cu', 'aoa_engine.cu', 'ensemble.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17', '-Xcompiler', '-fPIC']


def _nvcc() -> str:
    for cand in (shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found: the capb200 CUDA library cannot be built')


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = True) -> str:
    nvcc = _nvcc()
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    headers.append(os.path.join(os.path.dirname(PKG), 'include', 'capb200.h'))

    def compile_one(src):
        obj = os.path.join(OBJ, src.replace('.cu', '.o'))
        srcp = os.path.join(CSRC, src)
        if force or _stale(obj, [srcp] + headers):
            cmd = [nvcc] + NVCC_FLAGS + ['-c', srcp, '-o', obj]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (src, r.stdout, r.stderr))
            return obj, True
        return obj, False

    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        results = list(ex.map(compile_one, SOURCES))
    objs = [o for o, _ in results]
    if force or any(c for _, c in results) or _stale(LIB, objs):
        cmd = [nvcc, '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a']
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
        if verbose:
            print('built', LIB)
    return LIB


if __name__ == '__main__':
    build(force='--force' in sys.argv)
