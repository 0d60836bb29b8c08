"""The device-drawn StVD input front end (csrc/stvd.cu, vc_stvd_input_front_end), measured on the GPU:
  (a) device time of preprocess.input_front_end at bench size (B = 1, 2, 4 scenes of 16 k LiDAR + 400 k raw virtual points
      before the FOV cut), VirConv-T form (two streams, training: bin_num 2, shuffle) and VirConv-L form (fused), CUDA
      events over repeated calls, and the same body captured in a CUDA graph and replayed;
  (b) host-to-device upload of the collated cloud the front end takes (un-discarded) against the one the dataloader hands
      over today (discarded, masked), pinned memory, CUDA events;
  (c) host time (median of 7 runs after a warm-up) of the numpy work the dataloader no longer runs per batch: split, input_point_discard (oracle/stvd.py, the
      reference's statements), mask_points_by_range and the shuffle of both streams;
  (d) the captured VirConv-T (VirConv8x, bf16) training step at 2 scenes of the same size, 16 000 voxels per stream: the
      front end inside the graph (the un-discarded cloud uploaded) against outside it (the split, discarded cloud of (c)
      uploaded, voxelisers in the graph), alternating, min over rounds of CUDA-event step times.
Prints the device name and power limit with the numbers.

    python profiles/microbench_input_front_end.py [--reps 50]
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

from oracle import stvd as o_stvd                                          # noqa: E402
from virconv_b200 import preprocess, scenes                               # noqa: E402

DEV = torch.device('cuda:0')
PC = np.array(scenes.POINT_CLOUD_RANGE, dtype=np.float32)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'nvidia-smi unavailable'
    return f'{torch.cuda.get_device_name(DEV)} | {q}'


def events(fn, reps):
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps


def frames(B):
    return [scenes.make_points(3 + b, 16384, 400000) for b in range(B)]


def collate(clouds):
    return np.ascontiguousarray(np.concatenate([np.pad(p, ((0, 0), (1, 0)), constant_values=b) for b, p in enumerate(clouds)]))


def host_flow(clouds, later_fusion=True):
    """The per-frame numpy work the front end replaces (dataset.py:270-298, data_processor.py:76-124)."""
    out = []
    for p in clouds:
        mm = p[p[:, -1] == 1]
        lidar = p[p[:, -1] == 2]
        kept = o_stvd.input_point_discard(mm, bin_num=2, rate=0.8)
        streams = [lidar, kept] if later_fusion else [np.concatenate([lidar, kept])]
        res = []
        for s in streams:
            s = s[(s[:, 0] >= PC[0]) & (s[:, 0] <= PC[3]) & (s[:, 1] >= PC[1]) & (s[:, 1] <= PC[4])]
            res.append(s[np.random.permutation(s.shape[0])])
        out.append(res)
    return out


def captured_step(reps, rounds=3):
    from oracle.testing import fill_module
    from virconv_b200.backbone import VirConv8x
    from virconv_b200.graph import GraphedStep, masked_mean
    cfg = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.15, NUM_FILTERS=[16, 32, 64, 64], MM=True)
    model = VirConv8x(cfg, 8, [1408, 1600, 80], precision='bf16')
    fill_module(model, 667)
    model = model.to(DEV).train()

    def loss_fn(out):
        ts = list(out['multi_scale_3d_features'].values()) + list(out['multi_scale_3d_features_mm'].values())
        return sum(masked_mean(t) for t in ts + [out['encoded_spconv_tensor']])
    pb = scenes.make_points_batch([3, 4], training=True, n_lidar=16384, n_virtual=400000)
    raw = torch.from_numpy(pb.points).pin_memory()
    split = host_flow([pb.points[pb.points[:, 0] == b][:, 1:] for b in range(2)])
    cat = lambda i: torch.from_numpy(np.concatenate([np.pad(f[i], ((0, 0), (1, 0)), constant_values=b)      # noqa: E731
                                                     for b, f in enumerate(split)])).pin_memory()
    base = dict(point_cloud_range=tuple(PC), voxel_size=(0.05, 0.05, 0.05), max_points_per_voxel=5, max_voxels=16000,
                vfe_model='max', max_voxels_mm=16000, vfe_model_mm=None)
    common = {'batch_size': 2, 'calib': pb.calib, 'aug_param': torch.from_numpy(pb.aug_param)}
    cases = {'inside': (dict(base, input_discard=dict(rate=0.8, later_fusion=True)), dict(common, points=raw)),
             'outside': (base, dict(common, points=cat(0), points_mm=cat(1)))}
    steps = {k: GraphedStep(model, loss_fn, margin=1.35, grain=1024, voxelizer=v) for k, (v, _) in cases.items()}
    for k, (_, batch) in cases.items():              # capture from device copies (the exact step reads them); time the uploads
        steps[k]({key: v.to(DEV) if key.startswith('points') else v for key, v in batch.items()})
    best = {k: float('inf') for k in cases}
    for _ in range(rounds):
        for k, (_, batch) in cases.items():
            best[k] = min(best[k], events(lambda: steps[k](batch), reps))
    print(f"(d) captured VirConv-T step, 2 scenes, host batch -> loss: front end inside {best['inside'] / 1e3:.3f} ms, "
          f"outside {best['outside'] / 1e3:.3f} ms per step (min of {rounds} alternating rounds of {reps})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    args = ap.parse_args()
    print('device:', card())
    for B in (1, 2, 4):
        clouds = frames(B)
        pts_h = torch.from_numpy(collate(clouds)).pin_memory()
        pts = pts_h.to(DEV)
        for later_fusion, label in ((True, 'VirConv-T form'), (False, 'VirConv-L form')):
            fn = lambda: preprocess.input_front_end(pts, B, True, later_fusion, static=True)      # noqa: E731
            t_eager = events(fn, args.reps)
            g = torch.cuda.CUDAGraph()
            fn()
            torch.cuda.synchronize()
            with torch.cuda.graph(g):
                out = fn()
            t_graph = events(g.replay, args.reps)
            torch.cuda.synchronize()
            rows = [int(out[k].num_rows) for k in ('points', 'points_mm') if k in out]
            print(f'(a) B={B} {label}: {pts.shape[0]} input rows -> {rows} rows; front end {t_eager:.1f} us per call eager, '
                  f'{t_graph:.1f} us per replay captured')
        discarded = host_flow(clouds)                  # (warm-up)
        times = []
        for _ in range(7):
            t0 = time.perf_counter()
            host_flow(clouds)
            times.append((time.perf_counter() - t0) * 1e3)
        t_host = float(np.median(times))
        small_h = torch.from_numpy(np.concatenate([np.concatenate(s) for s in discarded])).pin_memory()
        big_d, small_d = torch.empty_like(pts), torch.empty(small_h.shape, dtype=torch.float32, device=DEV)
        t_big = events(lambda: big_d.copy_(pts_h, non_blocking=True), args.reps)
        t_small = events(lambda: small_d.copy_(small_h, non_blocking=True), args.reps)
        print(f'(b) B={B} upload: un-discarded {pts_h.shape[0]} rows {t_big:.1f} us, discarded {small_h.shape[0]} rows '
              f'{t_small:.1f} us')
        print(f'(c) B={B} host numpy split + discard + mask + shuffle: {t_host:.1f} ms per batch, median of 7 (one process)')
    captured_step(args.reps)


if __name__ == '__main__':
    main()
