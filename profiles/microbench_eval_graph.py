"""Test-time backbone forward, eager against CUDA-graph replay (graph.GraphedForward), at bench.py's eval workloads:
  T   VirConv-T, ROT_NUM = 3 (X_TRANS copies), batch 2, 16 k LiDAR + 80 k virtual points per scene, 40 000-voxel cap per stream
      and scene (VirConv-T.yaml test) — bench.py --model T's `eval_rot3`;
  L   VirConv-L eval forward, batch 2, the same scenes voxelised together, 40 000-voxel cap (bench.py --model L's batch).
Arms, alternated over several rounds, L2 flushed (256 MiB write) before every forward, bf16, under torch.no_grad():
  eager       the eval forward as the detector calls it (exact-shape plan executor; VirConv-T: torch.cat of the copies, host
              reads of the strided convs' row counts, torch.nonzero per split tensor and copy, one MM plan call per copy);
  graph       GraphedForward over the voxelised batch (voxel features / coordinates of every stream and copy copied in, one
              replay);
  graph+vox   GraphedForward with the in-graph voxelisers: the per-copy point clouds are the input.
Per-forward CUDA-event time (first enqueued work to last, host gaps included), host time per call, library launches per
forward.  Prints the device name and power limit with the numbers.

    python profiles/microbench_eval_graph.py [--steps 30] [--rounds 5] [--models T,L]
"""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.testing import fill_module                                    # noqa: E402
from virconv_b200 import _lib, ops, scenes                                # noqa: E402
from virconv_b200.backbone import VirConv8x, VirConvL8x                   # noqa: E402
from virconv_b200.graph import GraphedForward                             # noqa: E402

CFG_T = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.15, NUM_FILTERS=[16, 32, 64, 64], MM=True)
CFG_L = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
N_LIDAR, N_VIRTUAL, MAX_VOXELS, ROT, POOL = 16384, 80000, 40000, 3, 2
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


def batches_t():
    vox, pts = [], []
    for i in range(POOL):
        ids = [100 + 2 * i, 101 + 2 * i]
        b = scenes.make_batch_mm(ids, N_LIDAR, N_VIRTUAL, MAX_VOXELS, training=False, rot_num=ROT)
        bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
        bd.update(batch_size=b.batch_size, calib=b.calib, transform_param=torch.from_numpy(b.transform_param.copy()))
        vox.append(bd)
        pd = {'batch_size': len(ids), 'calib': b.calib, 'transform_param': bd['transform_param']}
        clouds = {}
        for k, sid in enumerate(ids):
            raw = scenes.make_points(sid, N_LIDAR, N_VIRTUAL, scenes.Calib())
            for r in range(ROT):
                p = scenes.augment(raw, scenes.TEST_TRANSFORMS[r])
                s = '' if r == 0 else str(r)
                for key, ind in (('points', 2), ('points_mm', 1)):
                    q = scenes.mask_points_by_range(p[p[:, 7] == ind]).astype(np.float32)
                    clouds.setdefault(key + s, []).append(np.concatenate([np.full((q.shape[0], 1), k, np.float32), q], 1))
        pd.update({k: torch.from_numpy(np.concatenate(v)).to(DEV) for k, v in clouds.items()})
        pts.append(pd)
    return vox, pts


def batches_l():
    vox, pts = [], []
    for i in range(POOL):
        ids = [2 * i, 2 * i + 1]
        b = scenes.make_batch(ids, N_LIDAR, N_VIRTUAL, MAX_VOXELS, training=False)
        vox.append({'voxel_features': torch.from_numpy(b.voxel_features).to(DEV),
                    'voxel_coords': torch.from_numpy(b.voxel_coords).to(DEV), 'batch_size': b.batch_size, 'calib': b.calib})
        pb = scenes.make_points_batch(ids, N_LIDAR, N_VIRTUAL, training=False)
        pts.append({'points': torch.from_numpy(pb.points).to(DEV), 'batch_size': pb.batch_size, 'calib': pb.calib})
    return vox, pts


def run(name, model, vox_b, pts_b, args, lib, flush):
    def eager(bd):
        with torch.no_grad():
            return model(dict(bd))

    arms = {'eager': (eager, vox_b), 'graph': (GraphedForward(model, margin=MARGIN), vox_b),
            'graph+vox': (GraphedForward(model, margin=MARGIN, voxelizer=VOX), pts_b)}
    for _ in range(2):                                   # every batch through every arm (allocator pools, captures)
        for fn, bs in arms.values():
            for b in bs:
                fn(b)
    torch.cuda.synchronize()
    dev_ms = {k: [] for k in arms}
    host_ms = {k: [] for k in arms}
    launches = {}
    for _ in range(args.rounds):
        for arm, (fn, bs) in arms.items():
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
            launches[arm] = (lib.vc_launch_count() - l0) / args.steps
            torch.cuda.synchronize()
            dev_ms[arm].append(statistics.mean(a.elapsed_time(e) for a, e in evs))
            host_ms[arm].append(host * 1e3 / args.steps)
    assert int(ops.tc_error_flag(DEV).item()) == 0, 'tensor-core pipeline timeout flag set'
    print(f'{name}: {args.rounds} rounds x {args.steps} forwards, L2 flushed before each forward')
    for arm in arms:
        d, h = dev_ms[arm], host_ms[arm]
        extra = ''
        if arm != 'eager':
            g = arms[arm][0]
            extra = f'; library launches per replay {g.launches_per_replay}, re-captures {g.recaptures}'
        print(f'  {arm:10s} {statistics.median(d):7.3f} ms/forward device (median of rounds; min {min(d):.3f}, max {max(d):.3f}), '
              f'host {statistics.median(h):6.3f} ms/call, library launches enqueued by the host per forward {launches[arm]:.0f}'
              f'{extra}', flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--models', default='T,L')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    print('device:', card())
    lib = _lib.load()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=DEV)
    for m in args.models.split(','):
        if m == 'T':
            model = VirConv8x(CFG_T, 8, [1408, 1600, 80], precision='bf16')
            fill_module(model, 667)
            vox_b, pts_b = batches_t()
            n_l = statistics.mean(sum(b['voxel_features' + s].shape[0] for s in ('', '1', '2')) for b in vox_b)
            n_m = statistics.mean(sum(b['voxel_features_mm' + s].shape[0] for s in ('', '1', '2')) for b in vox_b)
            title = (f'VirConv-T eval forward, ROT_NUM=3, batch 2, {n_l:.0f} LiDAR + {n_m:.0f} virtual voxels over the 3 copies '
                     f'(mean of {POOL} batches), bf16')
        else:
            model = VirConvL8x(CFG_L, 8, [1408, 1600, 80], precision='bf16')
            fill_module(model, 666)
            vox_b, pts_b = batches_l()
            n = statistics.mean(b['voxel_features'].shape[0] for b in vox_b)
            title = f'VirConv-L eval forward, batch 2, {n:.0f} voxels (mean of {POOL} batches), bf16'
        run(title, model.to(DEV).eval(), vox_b, pts_b, args, lib, flush)
    print('device:', card())


if __name__ == '__main__':
    main()
