"""Part-score RoI pooling of TEDMHead's PART branch (VirConv-T / -S), two arms in one process on the same seeded inputs:
  reference — `TEDMHead.obtain_conf_preds` (ted_head.py:425-442) with `gen_sample_grid` and
              `bilinear_interpolate_torch_gridsample` (:110-156), its control flow restated over torch on the GPU: per
              scene the grid from `nonzero()` (one device-to-host read), the rotation of `rotate_points_along_z`, the
              normalisation, `F.grid_sample` over the 49 part channels and the mean; the backward is autograd's;
  fused     — virconv_b200.part_pool.part_pool (csrc/part_pool.cu), one launch forward, one backward.
Shapes: VirConv-T on KITTI, a [2, 49, 200, 176] part map (GRID_OFFSETS [0, 40], FEATMAP_STRIDE 0.4) with 2 x 160 RoIs
(a training stage) and 2 x 50 (a test-time stage, after NMS).  Times the forward (no grad) and forward + backward with
CUDA events over `--reps` calls, arms alternating, `--rounds` rounds after a warm-up; prints the median and the range
per call, the fused arm also replayed from a CUDA graph (its device time without the host's launch overhead), the largest
output differences between the arms, the algorithmic bytes of the fused kernels, and the device name and power limit.

    python profiles/microbench_part_pool.py [--reps 50] [--rounds 5]
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from virconv_b200.part_pool import part_pool       # noqa: E402

S = 7
OFFSETS = (0.0, 40.0)
SCALE = 1 / 0.4
MAP = (2, S * S, 200, 176)


def kitti_rois(B, N, seed, device):
    """car-sized RoIs over KITTI's point-cloud range (x in [0, 70.4], y in [-40, 40]), random headings, fp32"""
    rng = np.random.default_rng(seed)
    r = np.zeros((B, N, 7), np.float32)
    r[..., 0] = rng.uniform(-2.0, 72.0, (B, N))
    r[..., 1] = rng.uniform(-41.0, 41.0, (B, N))
    r[..., 2] = rng.uniform(-1.5, 0.0, (B, N))
    r[..., 3] = rng.uniform(3.2, 4.6, (B, N))
    r[..., 4] = rng.uniform(1.4, 1.9, (B, N))
    r[..., 5] = rng.uniform(1.3, 1.7, (B, N))
    r[..., 6] = rng.uniform(-np.pi, np.pi, (B, N))
    return torch.from_numpy(r).to(device)


def reference_arm(parts, rois, grid_size=S, grid_offsets=OFFSETS, spatial_scale=SCALE):
    confi = []
    for i in range(parts.shape[0]):
        boxes, im = rois[i], parts[i]
        N = boxes.shape[0]
        dense_idx = boxes.new_ones((grid_size, grid_size)).nonzero().repeat(N, 1, 1).float()
        size = boxes.view(N, -1)[:, 3:5]
        local = dense_idx / (grid_size - 1) * size.unsqueeze(dim=1) - (size.unsqueeze(dim=1) / 2)
        local = torch.cat([local, torch.ones_like(local[..., 0:1])], -1)
        angle = boxes[:, 6]
        cosa, sina = torch.cos(angle), torch.sin(angle)
        zeros, ones = angle.new_zeros(N), angle.new_ones(N)
        rot = torch.stack((cosa, sina, zeros, -sina, cosa, zeros, zeros, zeros, ones), dim=1).view(-1, 3, 3).float()
        pts = torch.matmul(local.clone()[:, :, 0:3], rot).squeeze(dim=1)
        pts = pts + boxes[:, 0:3].clone().unsqueeze(dim=1)
        x = (pts[..., 0:1].permute(1, 2, 0).contiguous() + grid_offsets[0]) * spatial_scale
        y = (pts[..., 1:2].permute(1, 2, 0).contiguous() + grid_offsets[1]) * spatial_scale
        xs, ys = x.view(grid_size ** 2, -1), y.view(grid_size ** 2, -1)
        C, H, W = im.shape
        samples = torch.cat([xs.unsqueeze(2).unsqueeze(3), ys.unsqueeze(2).unsqueeze(3)], 3)
        samples[:, :, :, 0] = samples[:, :, :, 0] / W
        samples[:, :, :, 1] = samples[:, :, :, 1] / H
        samples = samples * 2 - 1
        out = F.grid_sample(im.unsqueeze(1), samples, align_corners=False)
        confi.append(torch.mean(out, 0).view(-1, 1))
    return torch.cat(confi)


def fused_arm(parts, rois):
    return part_pool(parts, rois, S, OFFSETS, SCALE)


def time_arm(fn, parts, rois, g, backward, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        if backward:
            torch.autograd.grad(fn(parts, rois), [parts], g)
        else:
            with torch.no_grad():
                fn(parts, rois)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / reps * 1e3     # us per call


def graph_time(parts, rois, g, backward, reps):
    """the fused arm captured in a CUDA graph and replayed: the device time of its launches without the host's"""
    def step():
        if backward:
            return torch.autograd.grad(fused_arm(parts, rois), [parts], g)[0]
        with torch.no_grad():
            return fused_arm(parts, rois)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    graph.replay()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        graph.replay()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / reps * 1e3


def algorithmic_bytes(B, N, H, W):
    """fused forward: 4 taps x 49 parts of every RoI + the RoI rows + the output; backward: the whole dparts written
    + the RoI rows and g"""
    fwd = B * N * S * S * 4 * 4 + B * N * 7 * 4 + B * N * 4
    bwd = B * S * S * H * W * 4 + B * N * 7 * 4 + B * N * 4
    return fwd, bwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    dev = torch.device('cuda')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    print(f'device: {torch.cuda.get_device_name(0)} | nvidia-smi: {smi}')
    gen = torch.Generator(device=dev).manual_seed(0)
    parts = torch.randn(MAP, device=dev, generator=gen).requires_grad_()
    arms = (('reference', reference_arm), ('fused', fused_arm))
    for what, N in (('training stage, 2 x 160 RoIs', 160), ('test stage, 2 x 50 RoIs', 50)):
        rois = kitti_rois(MAP[0], N, 1 + N, dev)
        g = torch.randn((MAP[0] * N, 1), device=dev, generator=gen)
        res = {}
        for name, fn in arms:
            out = fn(parts, rois)
            (d,) = torch.autograd.grad(out, [parts], g)
            res[name] = (out.detach(), d)
        del out                                     # no autograd graph of `parts` may outlive this into a capture
        o_ref, d_ref = res['reference']
        o_fus, d_fus = res['fused']
        print(f'\n{what}: [2, 49, 200, 176] map')
        print(f'  agreement: out max |fused - reference| = {(o_fus - o_ref).abs().max().item():.3e} '
              f'(max |reference| {o_ref.abs().max().item():.3e}); dparts max diff = {(d_fus - d_ref).abs().max().item():.3e} '
              f'(max |reference| {d_ref.abs().max().item():.3e})')
        fb, bb = algorithmic_bytes(MAP[0], N, MAP[2], MAP[3])
        print(f'  fused algorithmic bytes: forward {fb / 1e3:.0f} KB, backward {bb / 1e6:.2f} MB')
        for backward in (False, True):
            for name, fn in arms:                   # warm-up
                time_arm(fn, parts, rois, g, backward, 5)
            t = {name: [] for name, _ in arms}
            for _ in range(args.rounds):
                for name, fn in arms:
                    t[name].append(time_arm(fn, parts, rois, g, backward, args.reps))
            label = 'forward + backward' if backward else 'forward (no grad)'
            for name, _ in arms:
                v = np.array(t[name])
                print(f'  {label:20s} {name:9s}: median {np.median(v):9.1f} us/call  (range {v.min():.1f}-{v.max():.1f}, '
                      f'{args.rounds} rounds x {args.reps})')
            print(f'  {label:20s} speed-up: {np.median(t["reference"]) / np.median(t["fused"]):.1f}x')
            v = np.array([graph_time(parts, rois, g, backward, args.reps * 4) for _ in range(args.rounds)])
            print(f'  {label:20s} fused, graph-replayed: median {np.median(v):.1f} us/call  (range {v.min():.1f}-'
                  f'{v.max():.1f}); {(fb + bb if backward else fb) / np.median(v) / 1e3:.0f} GB/s of algorithmic bytes')


if __name__ == '__main__':
    main()
