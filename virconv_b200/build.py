"""Build libvirconv_sm90.so (the C-ABI shared library of include/virconv_b200.h) in-tree with nvcc.

nvcc cross-compiles sm_90a without a GPU; the .so and the objects under lib/ are build products (git-ignored).
    python -m virconv_b200.build [--verbose] [--force]
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIBDIR = os.path.join(HERE, 'lib')
LIB = os.path.join(LIBDIR, 'libvirconv_sm90.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-O3', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo',
         '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr',
         '-DVC_BUILDING']
# per-source additions.  iou3d_nms.cu: no a*b+c contraction on either side, so that its __host__ __device__ box geometry
# rounds identically on the host (vc_boxes_iou_bev_host) and on the GPU
# anchor_targets.cu: no contraction either, so that its IoU and box encoding round every operation as torch's elementwise
# kernels do (the equality tests of the target assignment compare those values)
# roi_targets.cu: no contraction, so that the 3-D IoU it takes from box_geom.cuh is bit for bit vc_boxes_iou3d's and its
# labels round as torch's elementwise kernels do
# head_losses.cu: no contraction, so that each float64 operation of the losses and their gradients rounds once, as the
# float64 restatement in oracle/head_losses.py does
# part_pool.cu: no contraction, so that the sample positions and bilinear weights round every operation once, as torch's
# elementwise kernels and grid_sample do
# optim.cu: no contraction, so that every fp32 operation of the update rounds once, as torch's elementwise kernels do
# roi_grid.cu: no contraction, so that the grid points and their floor divisions round every operation once, as torch's
# elementwise kernels do
# box_decode.cu: no contraction, so that the decoded boxes, their rotations and the stage transforms round every
# operation once, as torch's elementwise kernels do
# kitti_eval.cu: no contraction, so that the overlaps round every operation once in the types numba gives the
# reference's kernels (kitti_eval_geom.cuh)
FILE_FLAGS = {'roi_grid.cu': ['-fmad=false', '-Xcompiler', '-ffp-contract=off'],'iou3d_nms.cu': ['-fmad=false', '-Xcompiler', '-ffp-contract=off'],
              'box_decode.cu': ['-fmad=false', '-Xcompiler', '-ffp-contract=off'],
              'optim.cu': ['-fmad=false', '-Xcompiler', '-ffp-contract=off'],
              'anchor_targets.cu': ['-fmad=false', '-Xcompiler', '-ffp-contract=off'],
              'roi_targets.cu': ['-fmad=false', '-Xcompiler', '-ffp-contract=off'],
              'head_losses.cu': ['-fmad=false', '-Xcompiler', '-ffp-contract=off'],
              'part_pool.cu': ['-fmad=false', '-Xcompiler', '-ffp-contract=off'],
              'kitti_eval.cu': ['-fmad=false', '-Xcompiler', '-ffp-contract=off']}


def flags_for(src):
    return FLAGS + FILE_FLAGS.get(os.path.basename(src), [])


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, 'rb') as f:
            h.update(p.encode())
            h.update(f.read())
    h.update(' '.join(FLAGS).encode())
    h.update(repr(sorted(FILE_FLAGS.items())).encode())
    return h.hexdigest()


def build(verbose: bool = False, force: bool = False, defines=(), suffix: str = '') -> str:
    """`defines` / `suffix`: debug variants (e.g. -DVC_TC_TRACE -> libvirconv_sm90_trace.so, picked up through the
    VIRCONV_LIB environment variable); the default build has neither."""
    os.makedirs(LIBDIR, exist_ok=True)
    if suffix:
        return _build_variant(list(defines), suffix, verbose)
    srcs = sources()
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))] + [
        os.path.join(os.path.dirname(HERE), 'include', 'virconv_b200.h')]
    stamp = os.path.join(LIBDIR, '.build_digest')
    dig = _digest(deps)
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    objs = []

    def compile_one(src):
        obj = os.path.join(LIBDIR, os.path.basename(src)[:-3] + '.o')
        cmd = [NVCC] + flags_for(src) + (['-Xptxas', '-v'] if verbose else []) + ['-c', src, '-o', obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (src, r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [NVCC, '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a', '-lcudart']
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    with open(stamp, 'w') as f:
        f.write(dig)
    return LIB


def _build_variant(defines, suffix, verbose):
    lib = os.path.join(LIBDIR, f'libvirconv_sm90_{suffix}.so')
    objs = []
    for src in sources():
        obj = os.path.join(LIBDIR, os.path.basename(src)[:-3] + f'_{suffix}.o')
        r = subprocess.run([NVCC] + flags_for(src) + [f'-D{d}' for d in defines] + ['-c', src, '-o', obj], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s' % (src, r.stderr))
        objs.append(obj)
    r = subprocess.run([NVCC, '-shared', '-o', lib] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a', '-lcudart'],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n' + r.stderr)
    return lib


if __name__ == '__main__':
    print(build(verbose='--verbose' in sys.argv, force='--force' in sys.argv))
