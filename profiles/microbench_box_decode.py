"""Device time and launches per call of the heads' box decoding and TEDMHead's cascade stage transforms: the reference's
control flow over torch (oracle/box_decode.py: decode_torch, limit_period, rotate_points_along_z's matmul, the per-scene
X_TRANS loops with their `if enable` host read) against the fused calls of virconv_b200.box_decode, on the same GPU.

  rpn    — AnchorHeadTemplate.generate_predicted_boxes' decode at VirConv-T size: 2 scenes x 70,400 anchors, 2 bins;
  rcnn   — RoIHeadTemplate.generate_predicted_boxes' decode at 2 x 160 RoIs;
  stages — the ROT_NUM = 3 stage-transform loop of an eval forward: pred_x_trans at every stage, roi_x_trans and
           roi_score_trans at stages 1 and 2, 2 x 160 boxes.

Device time: CUDA events around each call, with a 256 MB write between calls so that L2 starts cold; the median over
`--reps` calls per round, and the range over `--rounds` rounds, arms alternating.  Launches: the CUDA kernels and copies
torch.profiler records for one call.  The device name and power limit are printed beside the numbers.

    python profiles/microbench_box_decode.py [--reps 50] [--rounds 5]
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import box_decode as o  # noqa: E402
from virconv_b200 import box_decode as bd  # noqa: E402

B, A, N, R = 2, 70400, 160, 3
XT = [[0.3, 0.0, 0.98], [0.3, 1.0, 1.02], [0.0, 1.0, 1.0]]      # VirConv-T.yaml X_TRANS per stage


def kitti_anchors(dev):
    """VirConv-T's anchor layout: 200 x 176 locations (0.4 m) x rotations (0, 1.57), car size, bottom -1.78"""
    y, x = torch.meshgrid(torch.linspace(-40, 40, 200), torch.linspace(0, 70.4, 176), indexing='ij')
    a = torch.zeros(200, 176, 2, 7)
    a[..., 0], a[..., 1] = x[..., None], y[..., None]
    a[..., 2] = -1.78 + 1.56 / 2
    a[..., 3:6] = torch.tensor([3.9, 1.6, 1.56])
    a[..., 6] = torch.tensor([0.0, 1.57])
    return a.view(-1, 7).to(dev)


def kitti_rois(b, n, seed, dev, ld=7):
    gen = torch.Generator().manual_seed(seed)
    r = torch.zeros(b, n, ld)
    r[..., 0] = torch.rand(b, n, generator=gen) * 70
    r[..., 1] = torch.rand(b, n, generator=gen) * 80 - 40
    r[..., 2] = torch.rand(b, n, generator=gen) * 2 - 2
    r[..., 3] = 3 + torch.rand(b, n, generator=gen) * 1.5
    r[..., 4] = 1.4 + torch.rand(b, n, generator=gen) * 0.5
    r[..., 5] = 1.3 + torch.rand(b, n, generator=gen) * 0.4
    r[..., 6] = (torch.rand(b, n, generator=gen) * 2 - 1) * np.pi
    if ld > 7:
        r[..., 7:] = torch.rand(b, n, ld - 7, generator=gen)
    return r.to(dev)


def transform_param(dev):
    return torch.tensor([XT, XT], dtype=torch.float32, device=dev)


def stage_loop(arm, rois, preds, tp):
    """what multi_grid_pool_aggregation does with the stage transforms in eval, one set of RoIs / predictions"""
    x, s, p = ((o.torch_roi_x_trans, o.torch_roi_score_trans, o.torch_pred_x_trans) if arm == 'reference' else
               (lambda r, i, t: bd.roi_x_trans(_HEAD, r, i, t), lambda r, i, t: bd.roi_score_trans(_HEAD, r, i, t),
                lambda r, i, t: bd.pred_x_trans(_HEAD, r, i, t)))
    outs = []
    for i in range(R):
        if i >= 1:
            rois = x(rois, i, tp)
            outs.append(s(rois, i, tp))
        outs.append(p(preds, i, tp))
    return outs


class _XT:
    aug_config_list = [{'NAME': n} for n in bd.XTRANS_ORDER]


class _Head:
    x_trans_train = _XT()


_HEAD = _Head()


def workloads(dev):
    gen = torch.Generator(device=dev).manual_seed(5)
    anchors = kitti_anchors(dev)
    box = torch.randn(B, A, 7, device=dev, generator=gen) * 0.3
    dirs = torch.randn(B, A, 2, device=dev, generator=gen)
    rois = kitti_rois(B, N, 3, dev)
    rbox = torch.randn(B * N, 7, device=dev, generator=gen) * 0.3
    preds = kitti_rois(B, N, 4, dev)
    tp = transform_param(dev)
    return {
        'rpn': {'reference': lambda: o.torch_anchor_decode(box, anchors, dirs),
                'fused': lambda: bd.anchor_decode(box, anchors, dirs, 0.78539, 0.0, np.pi)},
        'rcnn': {'reference': lambda: o.torch_roi_decode(rbox, rois),
                 'fused': lambda: bd.roi_decode(rbox, rois)},
        'stages': {'reference': lambda: stage_loop('reference', rois, preds, tp),
                   'fused': lambda: stage_loop('fused', rois, preds, tp)},
    }


def launches(fn):
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def time_arm(fn, reps, flush):
    times = []
    for _ in range(reps):
        flush.fill_(1.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3)
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    dev = torch.device('cuda')
    torch.backends.cuda.matmul.allow_tf32 = False
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    print(f'device: {torch.cuda.get_device_name(0)} | nvidia-smi: {smi}')
    flush = torch.empty(64 << 20, device=dev)
    with torch.no_grad():
        for name, arms in workloads(dev).items():
            res = {arm: [] for arm in arms}
            for fn in arms.values():
                for _ in range(3):
                    fn()
            for _ in range(args.rounds):
                for arm, fn in arms.items():
                    res[arm].append(time_arm(fn, args.reps, flush))
            n = {arm: launches(fn) for arm, fn in arms.items()}
            line = ' | '.join(f'{arm}: {min(v):.1f}-{max(v):.1f} us, {n[arm]} launches' for arm, v in res.items())
            print(f'{name:7s} {line}')


if __name__ == '__main__':
    main()
