"""RoI target sampling of TEDMHead, two arms in one process on the same seeded inputs and the same uniforms:
  reference — `ProposalTargetLayer.forward` (proposal_target_layer.py:32-353) and the canonical transform of
              `RoIHeadTemplate.assign_targets` (roi_head_template.py:121-159), its control flow restated over torch on
              the GPU: per scene, the trimming loop reading one row sum per step, the per-class IoU with its `.item()` /
              `sum() > 0` reads and `nonzero()`, the three `nonzero()` of the subsampling, host draws copied to the
              device (oracle.roi_targets_golden.Draws, so both arms draw the same samples), then the labels and the
              transform as tensor ops; its 3-D IoU is this library's vc_boxes_iou3d, as reference_env binds it;
  fused     — virconv_b200.roi_targets.roi_targets_batched (csrc/roi_targets.cu).
Shapes: VirConv-L's STAGE0 (B = 2, 512 proposals -> 160) and the stage >= 1 shape (2 x 160 -> 160), 40 GT + 4 padding
rows per scene.  Reports synchronised host time per call, the largest output differences, and the device name and power
limit.

    python profiles/microbench_roi_targets.py [--reps 50]
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

from oracle import roi_targets_golden as g                                # noqa: E402
from virconv_b200 import iou3d_nms                                        # noqa: E402
from virconv_b200.reference_env import EasyDict                           # noqa: E402
from virconv_b200.roi_targets import SamplerConfig, empty_outputs, roi_targets_batched   # noqa: E402

N_GT = 40
KEYS = ('rois', 'gt_of_rois_src', 'gt_of_rois', 'gt_iou_of_rois', 'roi_scores', 'roi_labels', 'reg_valid_mask',
        'rcnn_cls_labels')


def scene(seed, B, M, G=N_GT + 4):
    rng = np.random.default_rng(seed)
    gt = np.zeros((B, G, 8), np.float32)
    rois = np.zeros((B, M, 7), np.float32)
    for b in range(B):
        rows = [g.gt_box(rng, 1) for _ in range(N_GT)]
        gt[b, :N_GT] = np.stack(rows)
        for i in range(M):
            rois[b, i] = g.near(rng, rows[rng.integers(N_GT)], rng.choice([0.1, 0.4, 1.0, 3.0])) if i % 8 else g.far(rng)
    return rois, rng.random((B, M)).astype(np.float32), np.ones((B, M), np.int64), gt


def _bg(hard, easy, n, draws, ratio, dev):
    if hard.numel() > 0 and easy.numel() > 0:
        h = min(int(n * ratio), len(hard))
        return torch.cat([hard[draws.torch_randint(0, hard.numel(), (h,)).to(dev)],
                          easy[draws.torch_randint(0, easy.numel(), (n - h,)).to(dev)]])
    src = hard if hard.numel() > 0 else easy
    return src[draws.torch_randint(0, src.numel(), (n,)).to(dev)]


def reference_targets(cfg, rois, scores, labels, gt, draws):
    """the reference's control flow over torch on the GPU (see the module docstring)"""
    dev = rois.device
    B, R = rois.shape[0], cfg.ROI_PER_IMAGE
    F = int(np.round(cfg.FG_RATIO * R))
    o_rois = rois.new_zeros(B, R, rois.shape[-1])
    o_gt = rois.new_zeros(B, R, gt.shape[-1])
    o_iou, o_scores = rois.new_zeros(B, R), rois.new_zeros(B, R)
    o_labels = rois.new_zeros((B, R), dtype=torch.long)
    for b in range(B):
        draws.new_scene()
        cur_gt = gt[b]
        k = len(cur_gt) - 1
        while k > 0 and cur_gt[k].sum() == 0:
            k -= 1
        cur_gt = cur_gt[:k + 1]
        gl = cur_gt[:, -1].long()
        ov = rois.new_zeros(rois.shape[1])
        asg = labels.new_zeros(rois.shape[1])
        for c in range(gl.min().item(), gl.max().item() + 1):
            rm, gm = labels[b] == c, gl == c
            if rm.sum() > 0 and gm.sum() > 0:
                mx, am = iou3d_nms.boxes_iou3d_gpu(rois[b][rm][:, :7], cur_gt[gm][:, :7]).max(dim=1)
                ov[rm] = mx
                asg[rm] = gm.nonzero().view(-1)[am]
        gcls = cur_gt[asg, -1]
        fg = torch.zeros_like(ov, dtype=torch.bool)
        hard = torch.zeros_like(fg)
        for i in range(len(cfg.REG_FG_THRESH)):
            m = gcls == (i + 1)
            fg |= (ov >= min(cfg.REG_FG_THRESH[i], cfg.CLS_FG_THRESH[i])) & m
            hard |= (ov < cfg.REG_FG_THRESH[i]) & (ov >= cfg.CLS_BG_THRESH_LO) & m
        fg, hard, easy = fg.nonzero().view(-1), hard.nonzero().view(-1), (ov < cfg.CLS_BG_THRESH_LO).nonzero().view(-1)
        nf, nb = fg.numel(), hard.numel() + easy.numel()
        if nf > 0 and nb > 0:
            kf = min(F, nf)
            sel = torch.cat([fg[torch.from_numpy(draws.permutation(nf)[:kf]).to(dev)],
                             _bg(hard, easy, R - kf, draws, cfg.HARD_BG_RATIO, dev)])
        elif nf > 0:
            sel = fg[torch.from_numpy(np.floor(draws.rand(R) * nf)).long().to(dev)]
        else:
            sel = _bg(hard, easy, R, draws, cfg.HARD_BG_RATIO, dev)
        o_rois[b], o_gt[b], o_iou[b] = rois[b][sel], cur_gt[asg[sel]], ov[sel]
        o_scores[b], o_labels[b] = scores[b][sel], labels[b][sel]
    gcls = o_gt[..., -1]
    reg = o_iou.new_zeros(o_iou.shape).long()
    cls = o_iou.new_zeros(o_iou.shape)
    for i in range(len(cfg.REG_FG_THRESH)):
        m = gcls == (i + 1)
        this = ((o_iou > cfg.REG_FG_THRESH[i]) & m).long()
        if cfg.ENABLE_HARD_SAMPLING:
            t = int(1 / cfg.HARD_SAMPLING_RATIO[i])
            prob = torch.zeros_like(m)
            prob[range(draws.np_randint(0, t), B, t)] = True
            this += ((o_iou < cfg.REG_FG_THRESH[i]) & (o_iou > cfg.HARD_SAMPLING_THRESH[i]) & m & prob).long()
        reg += this
        fgm, bgm = o_iou > cfg.CLS_FG_THRESH[i], o_iou < cfg.CLS_BG_THRESH[i]
        mid = ~fgm & ~bgm
        lab = fgm.float()
        lab[mid] = (o_iou[mid] - cfg.CLS_BG_THRESH[i]) / (cfg.CLS_FG_THRESH[i] - cfg.CLS_BG_THRESH[i])
        cls[m] = lab[m]
    src = o_gt.clone()
    ry = o_rois[..., 6] % (2 * np.pi)
    can = o_gt.clone()
    can[..., 0:3] -= o_rois[..., 0:3]
    can[..., 6] -= ry
    cosa, sina = torch.cos(-ry.view(-1)), torch.sin(-ry.view(-1))
    zeros, ones = torch.zeros_like(cosa), torch.ones_like(cosa)
    rot = torch.stack((cosa, sina, zeros, -sina, cosa, zeros, zeros, zeros, ones), 1).view(-1, 3, 3)
    pts = can.view(-1, 1, can.shape[-1])
    can = torch.cat((torch.matmul(pts[:, :, 0:3], rot), pts[:, :, 3:]), -1).view(B, R, -1)
    h = can[..., 6] % (2 * np.pi)
    opp = (h > np.pi * 0.5) & (h < np.pi * 1.5)
    h[opp] = (h[opp] + np.pi) % (2 * np.pi)
    h[h > np.pi] -= np.pi * 2
    can[..., 6] = torch.clamp(h, min=-np.pi / 2, max=np.pi / 2)
    return dict(zip(KEYS, (o_rois, src, can, o_iou, o_scores, o_labels, reg, cls)))


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
    cfg_d = EasyDict(g.CFG_L)
    cfg = SamplerConfig(cfg_d)
    for what, M in (('STAGE0, 2 x 512 -> 2 x 160', 512), ('stage >= 1, 2 x 160 -> 2 x 160', 160)):
        rois, scores, labels, gt = (torch.from_numpy(a).to(dev) for a in scene(M, 2, M))
        rng = np.random.default_rng(M + 1)
        u_host = (rng.random((2, max(M, cfg.R)), dtype=np.float32), rng.random((2, cfg.R), dtype=np.float32),
                  rng.random(cfg.n_cls, dtype=np.float32))
        u_dev = tuple(torch.from_numpy(u).to(dev) for u in u_host)
        out = empty_outputs(2, cfg.R, 7, 8, dev)
        ref = reference_targets(cfg_d, rois, scores, labels, gt, g.Draws(*u_host))
        roi_targets_batched(cfg, rois, scores, labels, gt, u_dev, out)
        torch.cuda.synchronize()
        exact = all(torch.equal(ref[k], out[k]) for k in ('rois', 'gt_of_rois_src', 'roi_scores', 'roi_labels',
                                                          'reg_valid_mask'))
        d_iou = float((ref['gt_iou_of_rois'] - out['gt_iou_of_rois']).abs().max())
        d_cls = float((ref['rcnn_cls_labels'] - out['rcnn_cls_labels']).abs().max())
        d_can = float((ref['gt_of_rois'] - out['gt_of_rois']).abs().max())
        t_ref = _time(lambda: reference_targets(cfg_d, rois, scores, labels, gt, g.Draws(*u_host)), args.reps)
        t_new = _time(lambda: roi_targets_batched(cfg, rois, scores, labels, gt, u_dev, out), args.reps)
        print(f'{what}: reference {t_ref:.3f} ms, fused {t_new:.3f} ms; sampled rows / gathered GT / scores / labels / '
              f'reg_valid_mask identical: {exact}; max |diff| gt_iou {d_iou:.2e}, rcnn_cls_labels {d_cls:.2e}, '
              f'gt_of_rois {d_can:.2e}; reg_valid {int(out["reg_valid_mask"].sum())}')
    print(f'times: synchronised host time per call, {args.reps} repetitions after 3 warm-up calls')


if __name__ == '__main__':
    main()
