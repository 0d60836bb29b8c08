"""Build oracle/_ref/libiou3d_nms_ref.so: the REFERENCE's own rotated-box IoU / NMS kernels
(pcdet/ops/iou3d_nms/src/iou3d_nms_kernel.cu, stand-alone: it includes only <stdio.h>), compiled for sm_90a from where the
source lies — nothing is copied — together with oracle/csrc/iou3d_ref_shim.cu (C-linkage doors, and the reference's host
side of nms_gpu).  TEST INFRASTRUCTURE (see oracle/__init__.py), the companion of oracle/ref_build.py.  The library is
git-ignored and travels to the GPU machine with the working tree; it is read by oracle/iou3d_golden.py (which records the
fixtures under tests/golden) and by profiles/microbench_iou3d_nms.py.

    python -m oracle.iou3d_ref_build
"""
from __future__ import annotations

import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = '/root/reference/pcdet/ops/iou3d_nms/src'
OUT_DIR = os.path.join(HERE, '_ref')
LIB = os.path.join(OUT_DIR, 'libiou3d_nms_ref.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')


def available() -> bool:
    return os.path.exists(LIB)


def build(force: bool = False):
    """-> path of the library, or None when the reference sources are absent (GPU machine: the prebuilt file, if it
    travelled)."""
    if not os.path.isdir(REF_SRC):
        return LIB if available() else None
    srcs = [os.path.join(HERE, 'csrc', 'iou3d_ref_shim.cu'), os.path.join(REF_SRC, 'iou3d_nms_kernel.cu')]
    if available() and not force and all(os.path.getmtime(LIB) >= os.path.getmtime(s) for s in srcs):
        return LIB
    os.makedirs(OUT_DIR, exist_ok=True)
    cmd = [NVCC, '-O3', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '-shared', '-Xcompiler', '-fPIC',
           '-o', LIB] + srcs
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('building the reference iou3d_nms kernels failed:\n%s\n%s' % (r.stdout, r.stderr))
    return LIB


if __name__ == '__main__':
    print(build(force=True))
