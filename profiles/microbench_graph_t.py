"""VirConv-T / VirConv-S training step (VirConv8x: LiDAR stream + virtual-point stream) eager against CUDA-graph replay, at
bench.py's T training workload: batch 2, 16 k LiDAR + 80 k virtual points per scene, 16 000-voxel cap per stream and scene,
bf16, loss = sum of the masked means of the nine published tensors, L2 flushed (256 MiB write) before every step.
  eager       exact-shape executor path: two vc_exec_forward calls per step, host reads of the data-dependent row counts,
              Python autograd between them;
  graph       graph.GraphedStep over the voxelised batch (voxel features / coordinates of both streams copied into the
              graph's input buffers, then one replay);
  graph+vox   graph.GraphedStep with the in-graph voxelisers: the collated `points` / `points_mm` are the step's input, two
              vc_voxelize_mean calls run inside the graph.
Per-step CUDA-event time (device time from the step's first enqueued work to its last, host gaps included) and host time
per call, alternating the arms over several rounds; library launches per step; re-captures.  Prints the device name and
power limit with the numbers.

    python profiles/microbench_graph_t.py [--steps 40] [--rounds 5]
"""
from __future__ import annotations

import argparse
import copy
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.testing import fill_module                                    # noqa: E402
from virconv_b200 import _lib, ops, scenes                                # noqa: E402
from virconv_b200.backbone import VirConv8x                               # noqa: E402
from virconv_b200.graph import GraphedStep, masked_mean                   # noqa: E402

CFG_T = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.15, NUM_FILTERS=[16, 32, 64, 64], MM=True)
N_LIDAR, N_VIRTUAL, MAX_VOXELS, POOL = 16384, 80000, 16000, 4
VOX = dict(point_cloud_range=(0, -40, -3, 70.4, 40, 1), voxel_size=(0.05, 0.05, 0.05), max_points_per_voxel=5,
           max_voxels=MAX_VOXELS, vfe_model='max', max_voxels_mm=MAX_VOXELS, vfe_model_mm=None)
MARGIN = 1.15                                                             # bench.py's default capacity head-room
DEV = torch.device('cuda:0')


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'nvidia-smi unavailable'
    return f'{torch.cuda.get_device_name(DEV)} | {q}'


def loss_of(out):
    named = [out['encoded_spconv_tensor']] + [t for g in ('multi_scale_3d_features', 'multi_scale_3d_features_mm')
                                              for t in out[g].values()]
    return sum(masked_mean(t) for t in named)


def batches():
    vox, pts = [], []
    for i in range(POOL):
        ids = [2 * i, 2 * i + 1]
        b = scenes.make_batch_mm(ids, N_LIDAR, N_VIRTUAL, MAX_VOXELS, training=True)
        bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
        bd.update(batch_size=b.batch_size, calib=b.calib, aug_param=torch.from_numpy(b.aug_param))
        vox.append(bd)
        pb = scenes.make_points_batch(ids, N_LIDAR, N_VIRTUAL, training=True)
        p = torch.from_numpy(pb.points)
        pts.append({'points': p[p[:, 8] == 2].contiguous().to(DEV), 'points_mm': p[p[:, 8] == 1].contiguous().to(DEV),
                    'batch_size': pb.batch_size, 'calib': pb.calib, 'aug_param': torch.from_numpy(pb.aug_param)})
    return vox, pts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    print('device:', card())
    lib = _lib.load()
    vox_b, pts_b = batches()
    base = VirConv8x(CFG_T, 8, [1408, 1600, 80], precision='bf16')
    fill_module(base, 667)
    base.to(DEV).train()
    models = {k: copy.deepcopy(base) for k in ('eager', 'graph', 'graph+vox')}

    def eager(bd):
        m = models['eager']
        for p in m.parameters():
            p.grad = None
        loss = loss_of(m(dict(bd)))
        loss.backward()
        return loss

    g_vox = GraphedStep(models['graph'], loss_of, margin=MARGIN)
    g_pts = GraphedStep(models['graph+vox'], loss_of, margin=MARGIN, voxelizer=VOX)
    arms = {'eager': (eager, vox_b), 'graph': (g_vox, vox_b), 'graph+vox': (g_pts, pts_b)}
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=DEV)

    # same batch, same weights: the three arms compute the same loss (a captured step against the exact one)
    check = {k: float(fn(bs[0]).detach()) for k, (fn, bs) in arms.items()}
    print('loss of batch 0: ' + ', '.join(f'{k} {v:.7f}' for k, v in check.items()))
    for _ in range(2):                                   # every batch through every arm (allocator pools, captures)
        for fn, bs in arms.values():
            for b in bs:
                fn(b)
    torch.cuda.synchronize()
    dev_ms = {k: [] for k in arms}
    host_ms = {k: [] for k in arms}
    launches = {}
    for _ in range(args.rounds):                         # alternate the arms
        for name, (fn, bs) in arms.items():
            torch.cuda.synchronize()
            evs, host = [], 0.0
            l0 = lib.vc_launch_count()
            for s in range(args.steps):
                flush.zero_()
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                t0 = time.perf_counter()
                fn(bs[s % POOL])
                host += time.perf_counter() - t0
                e.record()
                evs.append((a, e))
            launches[name] = (lib.vc_launch_count() - l0) / args.steps
            torch.cuda.synchronize()
            dev_ms[name].append(statistics.mean(a.elapsed_time(e) for a, e in evs))
            host_ms[name].append(host * 1e3 / args.steps)
    assert int(ops.tc_error_flag(DEV).item()) == 0, 'tensor-core pipeline timeout flag set'
    n_l = sum(b['voxel_features'].shape[0] for b in vox_b) / POOL
    n_m = sum(b['voxel_features_mm'].shape[0] for b in vox_b) / POOL
    print(f'VirConv8x bf16 training step, batch 2, {n_l:.0f} LiDAR + {n_m:.0f} virtual voxels per batch (mean of {POOL}), '
          f'{args.rounds} rounds x {args.steps} steps, L2 flushed before each step')
    for name in arms:
        d, h = dev_ms[name], host_ms[name]
        extra = ''
        if name != 'eager':
            g = arms[name][0]
            extra = f'; library launches per replay {g.launches_per_replay}, re-captures {g.recaptures}'
        print(f'  {name:10s} {statistics.median(d):7.3f} ms/step device (median of rounds; min {min(d):.3f}, max {max(d):.3f}), '
              f'host {statistics.median(h):6.3f} ms/call, library launches enqueued by the host per step {launches[name]:.0f}'
              f'{extra}')
    print('device:', card())


if __name__ == '__main__':
    main()
