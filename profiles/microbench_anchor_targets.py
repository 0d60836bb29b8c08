"""RPN anchor mask and target assignment of AnchorHeadSingle, two arms in one process on the same seeded inputs:
  reference — `AnchorHeadSingle.get_anchor_mask` (anchor_head_single.py:75-115) and
              `AxisAlignedTargetAssigner.assign_targets` (axis_aligned_target_assigner.py:46-243) restated statement for
              statement over torch on the GPU: per scene and per anchor set, with the host copies of the IoU matrix for
              its argmaxes, the class mask through the host and the `nonzero()` calls;
  fused     — virconv_b200.anchor_targets.anchor_mask / AxisAlignedTargetAssigner (csrc/anchor_targets.cu).
Inputs: VirConv-L's anchor config (200 x 176 map, 2 rotations), the points of scenes.make_points_batch at bench.py's
scene sizes, B = 2, 40 car boxes per scene plus zero padding.  The targets run on the masked anchors (what the head
passes) and on the whole map.  The reference's mask indexes CPU tensors with CUDA index tensors, which torch 2.11
accepts (through a host round trip).  Reports synchronised host time per call, the largest output difference, and the
device name and power limit.

    python profiles/microbench_anchor_targets.py [--reps 50]
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import anchor_targets as o                                    # noqa: E402
from oracle import anchor_targets_golden as g                             # noqa: E402
from virconv_b200 import scenes                                           # noqa: E402
from virconv_b200.anchor_targets import AxisAlignedTargetAssigner, anchor_mask   # noqa: E402

N_LIDAR, N_VIRTUAL = 16384, 80000                                         # bench.py's scene sizes
N_GT = 40


def reference_mask(points, shape, voxel_size, pc_range):
    """get_anchor_mask, statement for statement (returns a CPU bool mask, as the reference does)"""
    stride = np.round(voxel_size * 8. * 10.)
    minx, miny = pc_range[0], pc_range[1]
    mask = torch.zeros(shape[-2], shape[-1])
    mask_large = torch.zeros(shape[-2] // 10, shape[-1] // 10)
    in_x = (points[:, 1] - minx) / stride
    in_y = (points[:, 2] - miny) / stride
    in_x = in_x.long().clamp(max=shape[-1] // 10 - 1)
    in_y = in_y.long().clamp(max=shape[-2] // 10 - 1)
    mask_large[in_y, in_x] = 1
    mask_large = mask_large.clone().int().detach().cpu().numpy()
    mask_large_index = np.argwhere(mask_large > 0) * 10
    index_list = []
    for i in np.arange(-10, 10, 1):
        for j in np.arange(-10, 10, 1):
            index_list.append(mask_large_index + [i, j])
    inds = torch.from_numpy(np.concatenate(index_list, 0)).cuda().long()
    mask[inds[:, 0], inds[:, 1]] = 1
    return mask.bool()


def _limit_period(val, offset=0.5, period=np.pi):
    return val - torch.floor(val / period + offset) * period


def _nearest_bev_iou(a, b):
    def bev(boxes):
        rot = _limit_period(boxes[:, 6]).abs()
        d = torch.where(rot[:, None] < np.pi / 4, boxes[:, [3, 4]], boxes[:, [4, 3]])
        return torch.cat((boxes[:, 0:2] - d / 2, boxes[:, 0:2] + d / 2), dim=1)
    ba, bb = bev(a), bev(b)
    x_min = torch.max(ba[:, 0, None], bb[None, :, 0])
    x_max = torch.min(ba[:, 2, None], bb[None, :, 2])
    y_min = torch.max(ba[:, 1, None], bb[None, :, 1])
    y_max = torch.min(ba[:, 3, None], bb[None, :, 3])
    x_len = torch.clamp_min(x_max - x_min, min=0)
    y_len = torch.clamp_min(y_max - y_min, min=0)
    area_a = (ba[:, 2] - ba[:, 0]) * (ba[:, 3] - ba[:, 1])
    area_b = (bb[:, 2] - bb[:, 0]) * (bb[:, 3] - bb[:, 1])
    inter = x_len * y_len
    return inter / torch.clamp_min(area_a[:, None] + area_b[None, :] - inter, min=1e-6)


def _encode(boxes, anchors):
    anchors[:, 3:6] = torch.clamp_min(anchors[:, 3:6], min=1e-5)
    boxes[:, 3:6] = torch.clamp_min(boxes[:, 3:6], min=1e-5)
    xa, ya, za, dxa, dya, dza, ra = torch.split(anchors, 1, dim=-1)
    xg, yg, zg, dxg, dyg, dzg, rg = torch.split(boxes, 1, dim=-1)
    diagonal = torch.sqrt(dxa ** 2 + dya ** 2)
    return torch.cat([(xg - xa) / diagonal, (yg - ya) / diagonal, (zg - za) / dza, torch.log(dxg / dxa),
                      torch.log(dyg / dya), torch.log(dzg / dza), rg - ra], dim=-1)


def _single(anchors, gt_boxes, gt_classes, matched, unmatched):
    n = anchors.shape[0]
    dev = anchors.device
    labels = torch.ones((n,), dtype=torch.int32, device=dev) * -1
    ious = torch.zeros((n,), dtype=torch.float, device=dev) * -1
    if len(gt_boxes) > 0 and n > 0:
        ov = _nearest_bev_iou(anchors[:, 0:7], gt_boxes[:, 0:7])
        a2g = torch.from_numpy(ov.cpu().numpy().argmax(axis=1)).cuda()
        a2g_max = ov[torch.arange(n, device=dev), a2g]
        ious = a2g_max
        g2a = torch.from_numpy(ov.cpu().numpy().argmax(axis=0)).cuda()
        g2a_max = ov[g2a, torch.arange(gt_boxes.shape[0], device=dev)]
        g2a_max[g2a_max == 0] = -1
        forced = (ov == g2a_max).nonzero()[:, 0]
        force_gt = a2g[forced]
        labels[forced] = gt_classes[force_gt]
        pos = a2g_max >= matched
        labels[pos] = gt_classes[a2g[pos]]
        bg = (a2g_max < unmatched).nonzero()[:, 0]
        labels[bg] = 0
        labels[forced] = gt_classes[force_gt]
    else:
        labels[:] = 0
    fg = (labels > 0).nonzero()[:, 0]
    targets = anchors.new_zeros((n, 7))
    if len(gt_boxes) > 0 and n > 0:
        targets[fg, :] = _encode(gt_boxes[a2g[fg], :], anchors[fg, :])
    reg = anchors.new_zeros((n,))
    reg[labels > 0] = 1.0
    return labels, targets, reg, ious


def reference_assign(all_anchors, gt_with_classes, class_names, sets):
    """AxisAlignedTargetAssigner.assign_targets (not multihead), statement for statement"""
    names = np.array(class_names)
    gt_classes = gt_with_classes[:, :, -1]
    gt_boxes = gt_with_classes[:, :, :-1]
    outs = [[], [], [], []]
    for k in range(gt_with_classes.shape[0]):
        cur = gt_boxes[k]
        cnt = cur.__len__() - 1
        while cnt > 0 and cur[cnt].sum() == 0:
            cnt -= 1
        cur = cur[:cnt + 1]
        cur_cls = gt_classes[k][:cnt + 1].int()
        per = []
        for cfg, anchors in zip(sets, all_anchors):
            mask = torch.from_numpy(names[cur_cls.cpu() - 1] == cfg['class_name'])
            fm = anchors.shape[:2]
            per.append((fm, _single(anchors.view(-1, 7), cur[mask], cur_cls[mask], cfg['matched_threshold'],
                                    cfg['unmatched_threshold'])))
        for i in range(4):
            shape = (-1, 7) if i == 1 else (-1,)
            parts = [r[i].view(*fm, -1, 7) if i == 1 else r[i].view(*fm, -1) for fm, r in per]
            outs[i].append(torch.cat(parts, dim=-2 if i == 1 else -1).view(*shape))
    return [torch.stack(x, 0) for x in outs]


def _time(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    dev = torch.device('cuda:0')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    print(f'device: {torch.cuda.get_device_name(0)} | nvidia-smi: {smi}')
    pts = torch.from_numpy(scenes.make_points_batch([0, 1], N_LIDAR, N_VIRTUAL, training=True).points).to(dev)
    voxel_size = (g.PCR[3] - g.PCR[0]) / g.GRID[0]
    shape = g.FEATURE_SHAPE_L
    m_ref = reference_mask(pts, shape, voxel_size, g.PCR).to(dev)
    m_new = anchor_mask(pts, g.PCR, g.GRID, shape)
    R = args.reps
    t_ref = _time(lambda: reference_mask(pts, shape, voxel_size, g.PCR), R)
    t_new = _time(lambda: anchor_mask(pts, g.PCR, g.GRID, shape), R)
    print(f'anchor mask  ({pts.shape[0]} points, {int(m_new.sum())} of {m_new.numel()} cells): reference {t_ref:.3f} ms, '
          f'fused {t_new:.3f} ms, masks equal: {bool(torch.equal(m_ref, m_new))}')

    z = np.load(os.path.join(ROOT, 'tests', 'golden', 'anchor_targets_ref.npz'))
    anchors = torch.from_numpy(o.anchors_from_shifts(z['L.x_shifts0'], z['L.y_shifts0'], g.CAR['anchor_bottom_heights'],
                                                     g.CAR['anchor_sizes'], g.CAR['anchor_rotations'])).to(dev)
    rng = np.random.default_rng(0)
    loc = anchors.reshape(-1, 7)[:, :2][m_new.repeat_interleave(2).view(-1)].cpu().numpy()
    gt = np.zeros((2, N_GT + 8, 8), np.float32)
    for b in range(2):
        for j in range(N_GT):
            gt[b, j] = g.box(rng, loc[rng.integers(len(loc))] + rng.normal(0, 0.6, 2).astype(np.float32), 1)
    gt = torch.from_numpy(gt).to(dev)

    class Coder:
        code_size = 7
    assigner = AxisAlignedTargetAssigner(g.model_cfg([g.CAR]), ['Car'], Coder(), g.GRID, g.PCR)
    keys = ('box_cls_labels', 'box_reg_targets', 'reg_weights', 'gt_ious')
    for what, all_anchors in (('masked', [anchors[:, m_new]]), ('whole map', [anchors])):
        ref = reference_assign(all_anchors, gt, ['Car'], [g.CAR])
        new = assigner.assign_targets(all_anchors, gt)
        same = all(torch.equal(r, new[k]) for r, k in zip(ref, keys) if k != 'box_reg_targets')
        dt = float((ref[1] - new['box_reg_targets']).abs().max())
        t_ref = _time(lambda: reference_assign(all_anchors, gt, ['Car'], [g.CAR]), R)
        t_new = _time(lambda: assigner.assign_targets(all_anchors, gt), R)
        print(f'targets, {what} (B = 2 x {ref[0].shape[1]} anchors, {N_GT} GT + 8 padding rows): reference {t_ref:.3f} ms, '
              f'fused {t_new:.3f} ms; labels / reg_weights / gt_ious equal: {same}, max |target diff| {dt:.2e}')
    print(f'times: synchronised host time per call, {R} repetitions after 3 warm-up calls')


if __name__ == '__main__':
    main()
