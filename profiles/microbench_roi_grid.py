"""The front end of TEDMHead's voxel-RoI grid pooling over one VirConv-T training step, two arms in one process on the
same inputs and the same fused pool layers (virconv_b200.voxel_pool.NeighborVoxelSAModuleMSG):
  reference — oracle.roi_grid.reference_roi_grid_pool: the reference methods' control flow (ted_head.py:450-673) over
              torch — the grid from `nonzero()` (a device-to-host read), host-built constant tensors, per-scene loops, and
              a fresh voxel -> row map for every source of every call;
  fused     — virconv_b200.roi_grid.roi_grid_pool / roi_grid_pool_mm: one grid-point launch per call, one map and one set
              of voxel centres per published tensor and batch_dict.
The step: 3 stages x (the G = 6 LiDAR branch + the G = 4 MM branch) x {x_conv3, x_conv4}, each stage calling both
branches with i = 0 as VirConv-T's training forward does (ted_head.py:794-795), in a new batch_dict per step.  Inputs:
the x_conv3 / x_conv4 tensors a VirConvL8x forward publishes on scenes.make_batch at bench.py's scene sizes (scenes 0, 1
for the LiDAR branch, 2, 3 for the MM branch; VirConv8x publishes the same shapes), 2 x 160 car-sized RoIs per stage.
The pool layers run forward only (no_grad), in training mode.  Reports per step, arms alternating over --rounds rounds:
host time ending in a synchronise, device time from CUDA events, the peak-memory increase, the largest output
difference between the arms, and the device name and power limit.

    python profiles/microbench_roi_grid.py [--reps 20] [--rounds 5]
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'profiles'))

from microbench_part_pool import kitti_rois                    # noqa: E402
from microbench_voxel_pool import CFG, LAYERS, MAX_VOXELS, N_LIDAR, N_VIRTUAL, PCR, VS   # noqa: E402
from oracle.roi_grid import reference_roi_grid_pool            # noqa: E402
from virconv_b200 import roi_grid, scenes                      # noqa: E402
from virconv_b200.backbone import VirConvL8x                   # noqa: E402
from virconv_b200.voxel_pool import NeighborVoxelSAModuleMSG   # noqa: E402

SOURCES = ('x_conv3', 'x_conv4')
STAGES = 3


def published(dev):
    torch.manual_seed(666)
    model = VirConvL8x(CFG, 8, [1408, 1600, 80]).to(dev).train()
    out = []
    for ids in ([0, 1], [2, 3]):
        b = scenes.make_batch(ids, N_LIDAR, N_VIRTUAL, MAX_VOXELS, training=True)
        bd = {'voxel_features': torch.from_numpy(b.voxel_features).to(dev),
              'voxel_coords': torch.from_numpy(b.voxel_coords).to(dev), 'batch_size': b.batch_size, 'calib': b.calib,
              'aug_param': torch.from_numpy(b.aug_param)}
        with torch.no_grad():
            out.append({s: model(bd)['multi_scale_3d_features'][s] for s in SOURCES})
    return out


def make_head(c_in, dev):
    torch.manual_seed(7)
    layers = lambda: torch.nn.ModuleList([NeighborVoxelSAModuleMSG(   # noqa: E731
        query_ranges=LAYERS[s]['query_ranges'], radii=LAYERS[s]['radii'], nsamples=[16, 16],
        mlps=[[c_in, 32, 32], [c_in, 32, 32]]) for s in SOURCES]).to(dev).train()
    ns = types.SimpleNamespace
    return ns(pool_cfg=ns(GRID_SIZE=6, FEATURES_SOURCE=list(SOURCES)),
              pool_cfg_mm=ns(GRID_SIZE=4, FEATURES_SOURCE=list(SOURCES)), roi_grid_pool_layers=layers(),
              roi_grid_pool_layers_mm=layers(), point_cloud_range=PCR, voxel_size=[float(v) for v in VS])


def step_fn(arm, head, lidar, mm, rois):
    def step():
        bd = {'batch_size': 2, 'multi_scale_3d_features': lidar, 'multi_scale_3d_features_mm': mm,
              'multi_scale_3d_strides': {s: LAYERS[s]['stride'] for s in SOURCES}}
        outs = []
        with torch.no_grad():
            for r in rois:
                bd['rois'] = r
                if arm == 'reference':
                    outs += [reference_roi_grid_pool(head, bd, 0), reference_roi_grid_pool(head, bd, 0, mm=True)]
                else:
                    outs += [roi_grid.roi_grid_pool(head, bd, 0), roi_grid.roi_grid_pool_mm(head, bd, 0)]
        return outs
    return step


def time_arm(fn, reps):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps, e0.elapsed_time(e1) / reps


def peak(fn):
    fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    a = ap.parse_args()
    dev = torch.device('cuda')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    print(f'device: {torch.cuda.get_device_name(0)} | nvidia-smi: {smi}')
    lidar, mm = published(dev)
    print('published rows:', {s: (lidar[s].features.shape[0], mm[s].features.shape[0]) for s in SOURCES},
          'channels', lidar['x_conv3'].features.shape[1])
    head = make_head(lidar['x_conv3'].features.shape[1], dev)
    rois = [kitti_rois(2, 160, 31 + k, dev) for k in range(STAGES)]
    arms = {name: step_fn(name, head, lidar, mm, rois) for name in ('reference', 'fused')}
    # same outputs: the pool layers are in training mode, so compare one eval-mode pass (running stats untouched)
    for m in list(head.roi_grid_pool_layers) + list(head.roi_grid_pool_layers_mm):
        m.eval()
    ref, fused = arms['reference'](), arms['fused']()
    diff = max(float((x - y).abs().max()) for x, y in zip(ref, fused))
    mag = max(float(x.abs().max()) for x in ref)
    print(f'largest output difference between the arms: {diff:.3g} (largest magnitude {mag:.3g})')
    for m in list(head.roi_grid_pool_layers) + list(head.roi_grid_pool_layers_mm):
        m.train()
    for fn in arms.values():
        for _ in range(3):
            fn()
    res = {k: [] for k in arms}
    for _ in range(a.rounds):
        for name, fn in arms.items():
            res[name].append(time_arm(fn, a.reps))
    for name in arms:
        host = [h for h, _ in res[name]]
        devt = [d for _, d in res[name]]
        print(f'{name:9s} per VirConv-T step ({STAGES} stages x 2 branches x 2 sources): host {np.median(host):.3f} ms '
              f'[{min(host):.3f}, {max(host):.3f}], device events {np.median(devt):.3f} ms [{min(devt):.3f}, {max(devt):.3f}], '
              f'peak +{peak(arms[name]):.1f} MiB')


if __name__ == '__main__':
    main()
