"""Rotated-box IoU / NMS: the reference's own kernels (oracle/_ref/libiou3d_nms_ref.so, with the host side of its nms_gpu:
per-scene mask, blocking copy to the host, CPU greedy) against csrc/iou3d_nms.cu (batched, device greedy), on the same
seeded inputs in one process, with the outputs compared.  Prints the device name and power limit beside the times.

    python profiles/microbench_iou3d_nms.py [--reps 50]
"""
from __future__ import annotations

import argparse
import ctypes
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import iou3d_golden as g          # noqa: E402
from oracle import iou3d_ref_build            # noqa: E402
from virconv_b200 import iou3d_nms            # noqa: E402


def _wall(fn, reps, warm=3):
    """host wall clock per call over `reps` calls ending in a device synchronise (the reference arm reads the host)"""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / reps * 1e3


def _events(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    assert iou3d_ref_build.available(), 'oracle/_ref/libiou3d_nms_ref.so missing: run __graft_entry__.build() where the reference is'
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    print(f'device: {torch.cuda.get_device_name(0)} | nvidia-smi: {smi}')
    lib = ctypes.CDLL(iou3d_ref_build.LIB)
    lib.ref_nms.restype = ctypes.c_int
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    R = args.reps

    print(f'{"case":34s} {"reference ms":>13s} {"new ms (wall)":>14s} {"new ms (events)":>16s}  agreement')
    for B, n, post, thresh in ((2, 4000, 512, 0.8), (2, 2000, 50, 0.75), (2, 4096, 500, 0.1)):
        boxes = np.stack([g.cars(n, 700 + b) for b in range(B)])
        sc = np.stack([g.scores(n, 800 + b) for b in range(B)])
        order = np.argsort(-sc, axis=1, kind='stable')
        sb = torch.from_numpy(np.ascontiguousarray(np.take_along_axis(boxes, order[..., None], 1))).cuda()
        keep_h = np.zeros(n, np.int64)

        def ref_arm():
            out = []
            for b in range(B):
                k = lib.ref_nms(p(sb[b]), n, ctypes.c_float(thresh), 0, keep_h.ctypes.data_as(ctypes.c_void_p))
                out.append(keep_h[:min(k, post)].copy())
            return out

        counts = torch.full((B,), n, dtype=torch.int32, device='cuda')
        new_arm = lambda: iou3d_nms._nms_sorted(sb, counts, thresh, post, False)
        t_ref = _wall(ref_arm, R)
        t_new = _wall(new_arm, R)
        t_ev = _events(new_arm, R)
        rk = ref_arm()
        keep, num = new_arm()
        keep, num = keep.cpu().numpy(), num.cpu().numpy()
        same = sum(int(np.array_equal(keep[b, :num[b]], rk[b])) for b in range(B))
        first = min(next((i for i in range(min(len(rk[b]), num[b])) if rk[b][i] != keep[b, i]), min(len(rk[b]), num[b]))
                    for b in range(B))
        print(f'{f"NMS B={B} x {n} -> {post} @ {thresh}":34s} {t_ref:13.3f} {t_new:14.3f} {t_ev:16.3f}  '
              f'keep lists identical {same}/{B} (kept {[int(x) for x in num]}'
              + (')' if same == B else f'; first difference at rank {first})'))

    for na, nb, what in ((512, 40, 'iou3d'), (4000, 4000, 'iou_bev')):
        a = torch.from_numpy(g.cars(na, 900)).cuda()
        b = torch.from_numpy(g.cars(nb, 901)).cuda() if what == 'iou3d' else a
        out = torch.zeros((na, nb), device='cuda')
        if what == 'iou3d':
            def ref_arm():
                # boxes_iou3d_gpu (iou3d_nms_utils.py:67-100): overlap kernel + torch glue
                ov = torch.zeros((na, nb), device='cuda')
                lib.ref_boxes_overlap_bev(na, p(a), nb, p(b), p(ov))
                a_max, a_min = (a[:, 2] + a[:, 5] / 2).view(-1, 1), (a[:, 2] - a[:, 5] / 2).view(-1, 1)
                b_max, b_min = (b[:, 2] + b[:, 5] / 2).view(1, -1), (b[:, 2] - b[:, 5] / 2).view(1, -1)
                oh = torch.clamp(torch.min(a_max, b_max) - torch.max(a_min, b_min), min=0)
                o3 = ov * oh
                va, vb = (a[:, 3] * a[:, 4] * a[:, 5]).view(-1, 1), (b[:, 3] * b[:, 4] * b[:, 5]).view(1, -1)
                return o3 / torch.clamp(va + vb - o3, min=1e-6)
            new_arm = lambda: iou3d_nms.boxes_iou3d_gpu(a, b)
        else:
            def ref_arm():
                lib.ref_boxes_iou_bev(na, p(a), nb, p(b), p(out))
                return out
            new_arm = lambda: iou3d_nms.boxes_iou_bev(a, b)
        t_ref = _events(ref_arm, R)
        t_new = _wall(new_arm, R)
        t_ev = _events(new_arm, R)
        d = float((ref_arm() - new_arm()).abs().max())
        print(f'{f"{what} {na} x {nb}":34s} {t_ref:13.3f} {t_new:14.3f} {t_ev:16.3f}  max |diff| {d:.2e}')
    print('reference ms: NMS = host wall clock (its host round trip included), IoU = CUDA events.')


if __name__ == '__main__':
    main()
