"""Seeded box generators of the rotated-box IoU / NMS tests, and the recorder of what the reference's own kernels
(oracle/_ref/libiou3d_nms_ref.so, built by oracle/iou3d_ref_build.py) return for them: tests/golden/iou3d_ref_iou.npz and
tests/golden/iou3d_ref_nms.npz.  Recording needs a GPU and the reference library; the fixtures are committed, so the tests
need neither.

    python -m oracle.iou3d_golden OUT_DIR
"""
from __future__ import annotations

import ctypes
import os
import sys

import numpy as np

NMS_SIZES = (1, 63, 64, 65, 2000, 4000)
NMS_THRESHOLDS = (0.1, 0.75, 0.8)
NEAR = 1e-4          # NMS cases keep no pair whose reference IoU lies this close to the threshold


def cars(n, seed, n_centres=30):
    """KITTI-like cars clustered around ~n_centres centres, as RPN output looks: (x, y, z, dx, dy, dz, heading) float32,
    dx 3.2-4.7, dy 1.4-1.9, dz 1.4-1.7, heading U(-pi, pi)."""
    rng = np.random.default_rng(seed)
    k = max(1, min(n_centres, n // 4 or 1))
    centres = np.c_[rng.uniform(2, 68, k), rng.uniform(-38, 38, k)]
    which = rng.integers(0, k, n)
    xy = centres[which] + rng.normal(0, 0.8, (n, 2))
    z = rng.normal(-1.0, 0.2, n)
    return np.ascontiguousarray(np.c_[xy, z, rng.uniform(3.2, 4.7, n), rng.uniform(1.4, 1.9, n), rng.uniform(1.4, 1.7, n),
                                      rng.uniform(-np.pi, np.pi, n)].astype(np.float32))


def scores(n, seed):
    """distinct scores"""
    return (np.random.default_rng(seed).permutation(n).astype(np.float32) + 1) / (n + 1)


def edge_set():
    """hand-made degenerate and boundary cases around one car: identical boxes, 90 and 180 degree turns, nested boxes,
    shared edges, neighbours whose corners lie 5 mm outside (inside the 1 cm band), a 45 degree turn, headings across
    the +-pi branch cut, and zero-size boxes"""
    x, y, z, dx, dy, dz, h = 10.0, 5.0, -1.0, 4.0, 2.0, 1.5, 0.0
    rows = [
        (x, y, z, dx, dy, dz, h),
        (x, y, z, dx, dy, dz, h),                       # identical
        (x, y, z, dx, dy, dz, h + np.pi / 2),           # 90 degrees
        (x, y, z, dx, dy, dz, h + np.pi),               # 180 degrees
        (x, y, z, dx / 2, dy / 2, dz, h),               # nested
        (x + dx, y, z, dx, dy, dz, h),                  # shared short edge
        (x + dx / 2, y, z, dx, dy, dz, h),              # half overlap, long edges collinear
        (x, y + dy, z + 0.5, dx, dy, dz, h),            # shared long edge, shifted in z
        (x + dx + 0.005, y, z, dx, dy, dz, h),          # 5 mm gap: corners in the 1 cm band
        (x, y - dy - 0.005, z, dx, dy, dz, h),          # 5 mm gap on the other side
        (x, y, z, dx, dy, dz, np.pi / 4),               # 45 degrees
        (x + 0.5, y + 0.3, z, dx, dy, dz, np.pi - 1e-3),    # across the branch cut
        (x + 0.5, y + 0.3, z, dx, dy, dz, -np.pi + 1e-3),
        (x, y, z, 0.0, 0.0, 0.0, h),                    # zero-size
        (x + 1.0, y, z, 0.0, dy, dz, 0.3),              # zero length
        (x + 1.2, y - 0.4, z + 0.3, 3.9, 1.6, 1.5, 0.7),
    ]
    return np.asarray(rows, np.float32)


def iou_cases():
    """name -> (boxes_a, boxes_b)"""
    a = cars(512, 1)
    rng = np.random.default_rng(2)
    gt = a[rng.choice(512, 48, replace=False)].copy()
    gt[:, :2] += rng.normal(0, 0.3, (48, 2)).astype(np.float32)
    gt[:, 6] += rng.normal(0, 0.2, 48).astype(np.float32)
    c300 = cars(300, 3)
    e = edge_set()
    return {'rois512_gt48': (a, gt), 'cars300': (c300, c300), 'edge': (e, e)}


def nms_boxes(n):
    return cars(n, 10 + n), scores(n, 20 + n)


def iou_normal_matrix(b):
    b = b.astype(np.float64)
    lo_x, hi_x = b[:, 0] - b[:, 3] / 2, b[:, 0] + b[:, 3] / 2
    lo_y, hi_y = b[:, 1] - b[:, 4] / 2, b[:, 1] + b[:, 4] / 2
    w = np.clip(np.minimum(hi_x[:, None], hi_x[None]) - np.maximum(lo_x[:, None], lo_x[None]), 0, None)
    h = np.clip(np.minimum(hi_y[:, None], hi_y[None]) - np.maximum(lo_y[:, None], lo_y[None]), 0, None)
    inter = w * h
    area = b[:, 3] * b[:, 4]
    return inter / np.maximum(area[:, None] + area[None] - inter, 1e-8)


def survivors(iou, thresh):
    """indices (into the sorted boxes) left after dropping, for every pair (i < j) whose IoU lies within NEAR of thresh,
    the later box unless one of the two is already gone (the IoU of the remaining pairs does not change)"""
    n = iou.shape[0]
    gone = np.zeros(n, bool)
    ii, jj = np.nonzero(np.triu(np.abs(iou - thresh) < NEAR, 1))
    for i, j in zip(ii, jj):
        if not (gone[i] or gone[j]):
            gone[j] = True
    return np.nonzero(~gone)[0]


def make(out_dir):
    import torch
    from oracle import iou3d_ref_build
    lib = ctypes.CDLL(iou3d_ref_build.LIB)
    lib.ref_nms.restype = ctypes.c_int
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    os.makedirs(out_dir, exist_ok=True)

    def ref_pair(fn, a, b):
        ta, tb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        out = torch.zeros((len(a), len(b)), device='cuda')
        torch.cuda.synchronize()
        getattr(lib, fn)(len(a), p(ta), len(b), p(tb), p(out))
        torch.cuda.synchronize()
        return out

    rec = {}
    for name, (a, b) in iou_cases().items():
        ov = ref_pair('ref_boxes_overlap_bev', a, b)
        rec[name + '_overlap'] = ov.cpu().numpy()
        rec[name + '_iou_bev'] = ref_pair('ref_boxes_iou_bev', a, b).cpu().numpy()
        # iou3d_nms_utils.boxes_iou3d_gpu :78-100 on the reference's overlaps
        ta, tb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        a_max, a_min = (ta[:, 2] + ta[:, 5] / 2).view(-1, 1), (ta[:, 2] - ta[:, 5] / 2).view(-1, 1)
        b_max, b_min = (tb[:, 2] + tb[:, 5] / 2).view(1, -1), (tb[:, 2] - tb[:, 5] / 2).view(1, -1)
        oh = torch.clamp(torch.min(a_max, b_max) - torch.max(a_min, b_min), min=0)
        o3 = ov * oh
        va, vb = (ta[:, 3] * ta[:, 4] * ta[:, 5]).view(-1, 1), (tb[:, 3] * tb[:, 4] * tb[:, 5]).view(1, -1)
        rec[name + '_iou3d'] = (o3 / torch.clamp(va + vb - o3, min=1e-6)).cpu().numpy()
    np.savez_compressed(os.path.join(out_dir, 'iou3d_ref_iou.npz'), **rec)

    nrec = {}
    for n in NMS_SIZES:
        boxes, sc = nms_boxes(n)
        order = np.argsort(-sc, kind='stable')
        sb = boxes[order]
        iou_rot = ref_pair('ref_boxes_iou_bev', sb, sb).cpu().numpy()
        iou_nrm = iou_normal_matrix(sb)
        for normal, iou in ((0, iou_rot), (1, iou_nrm)):
            for thresh in NMS_THRESHOLDS:
                keep_sorted = survivors(iou, thresh)          # indices into sb
                idx = np.sort(order[keep_sorted])             # surviving original indices
                b2, s2 = boxes[idx], sc[idx]
                o2 = np.argsort(-s2, kind='stable')
                tb = torch.from_numpy(np.ascontiguousarray(b2[o2])).cuda()
                keep = np.zeros(len(idx), np.int64)
                torch.cuda.synchronize()
                k = lib.ref_nms(p(tb), len(idx), ctypes.c_float(thresh), normal, keep.ctypes.data_as(ctypes.c_void_p))
                assert k >= 0
                key = f'{"normal" if normal else "rot"}_{n}_{thresh}'
                nrec[key + '_idx'] = idx.astype(np.int32)
                nrec[key + '_keep'] = o2[keep[:k]].astype(np.int32)     # = nms_gpu(b2, s2, thresh)[0]
    np.savez_compressed(os.path.join(out_dir, 'iou3d_ref_nms.npz'), **nrec)


if __name__ == '__main__':
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    make(sys.argv[1])
