"""Cost of the plan executor's deterministic mode (torch.use_deterministic_algorithms(True)), measured on the GPU:
  (a) bench.py's captured VirConvL8x bf16 training step (2 scenes x (16 k LiDAR + 80 k virtual), cap 40 000 voxels each):
      one GraphedStep captured with the flag off, one with it on, replayed alternately; min over rounds;
  (b) the eager VirConv-T (VirConv8x, MM) bf16 training step at the same size, flag off / on alternately;
  (c) the arena bytes the deterministic mode's partials, tables and operands take in one exact-mode VirConvL8x step.
Prints the device name and power limit with the numbers.

    python profiles/microbench_deterministic.py [--steps 40] [--rounds 5]
"""
from __future__ import annotations

import argparse
import copy
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.testing import fill_module                                    # noqa: E402
from virconv_b200 import executor, scenes                                 # noqa: E402
from virconv_b200.backbone import VirConv8x, VirConvL8x                   # noqa: E402
from virconv_b200.graph import GraphedStep, masked_mean                   # noqa: E402

CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG8 = dict(CFG, MM=True)
DEV = torch.device('cuda:0')


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'nvidia-smi unavailable'
    return f'{torch.cuda.get_device_name(DEV)} | {q}'


def batch(ids):
    b = scenes.make_batch(ids, 16384, 80000, 40000, training=True)
    return {'voxel_features': torch.from_numpy(b.voxel_features.copy()).to(DEV),
            'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).to(DEV), 'batch_size': 2, 'calib': b.calib,
            'aug_param': torch.from_numpy(b.aug_param.copy())}


def loss_of(out):
    named = dict(out['multi_scale_3d_features'])
    named['out'] = out['encoded_spconv_tensor']
    return sum(masked_mean(t) for t in named.values())


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for s in range(steps):
        fn(s)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def alternate(arms, steps, rounds):
    """arms: {name: (deterministic flag, fn(step index))} -> {name: [ms per step per round]}"""
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for name, (det, fn) in arms.items():
            torch.use_deterministic_algorithms(det)
            times[name].append(timed(fn, steps))
    torch.use_deterministic_algorithms(False)
    return times


def report(label, times, steps, rounds):
    for name, t in times.items():
        print(f'({label}) {name}: {min(t):.3f} ms/step (min of {rounds} rounds of {steps}; all: {", ".join(f"{v:.3f}" for v in t)})')


def graph_steps(steps, rounds):
    bs = [batch([2 * i, 2 * i + 1]) for i in range(2)]
    base = VirConvL8x(CFG, 8, [1408, 1600, 80], precision='bf16')
    fill_module(base, 666)
    base.to(DEV).train()
    arms = {}
    for name, det in (('flag off', False), ('flag on', True)):
        torch.use_deterministic_algorithms(det)
        g = GraphedStep(copy.deepcopy(base), loss_of, margin=1.15)
        for s in range(6):                           # exact-mode sizing run, capture, warm replays — all in this mode
            g(bs[s % 2])
        torch.cuda.synchronize()
        arms[name] = (det, lambda s, g=g: g(bs[s % 2]))
    times = alternate(arms, steps, rounds)
    print(f'(a) graph-replayed VirConvL8x bf16 step, {bs[0]["voxel_features"].shape[0]} input voxels:')
    report('a', times, steps, rounds)
    return base, bs[0]


def eager_t(steps, rounds):
    b = scenes.make_batch_mm([0, 1], n_lidar=16384, n_virtual=80000, max_voxels=40000, training=True)
    bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
    bd.update(batch_size=2, calib=b.calib, aug_param=torch.from_numpy(b.aug_param))
    m = VirConv8x(CFG8, 8, [1408, 1600, 80], precision='bf16')
    fill_module(m, 667)
    m.to(DEV).train()

    def one(_s):
        for p in m.parameters():
            p.grad = None
        out = m(dict(bd))
        pub = [t for g in ('multi_scale_3d_features', 'multi_scale_3d_features_mm') for t in out[g].values()]
        sum(masked_mean(t) for t in pub).backward()
    for det in (False, True, False, True):
        torch.use_deterministic_algorithms(det)
        one(0)
    times = alternate({'flag off': (False, one), 'flag on': (True, one)}, max(steps // 4, 5), rounds)
    print(f'(b) eager VirConv-T (VirConv8x, MM) bf16 step, {bd["voxel_features"].shape[0]} LiDAR + '
          f'{bd["voxel_features_mm"].shape[0]} virtual voxels:')
    report('b', times, max(steps // 4, 5), rounds)


def det_bytes(base, bd):
    runs = []
    note = executor.note_last_run
    executor.note_last_run = lambda model, run: (runs.append(run), note(model, run))
    try:
        m = copy.deepcopy(base)
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            loss_of(m(dict(bd))).backward()
            torch.cuda.synchronize()
            used = runs[-1].query(0, 0)[0]
            on, extra = runs[-1].deterministic_bytes()
            print(f'(c) exact-mode VirConvL8x bf16 step, deterministic {on}: arena {used / 2**20:.1f} MiB, of which the '
                  f'deterministic partials / tables / operands {extra / 2**20:.1f} MiB')
    finally:
        executor.note_last_run = note
        torch.use_deterministic_algorithms(False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    print('device:', card())
    base, bd = graph_steps(args.steps, args.rounds)
    eager_t(args.steps, args.rounds)
    det_bytes(base, bd)
    print('device:', card())


if __name__ == '__main__':
    main()
