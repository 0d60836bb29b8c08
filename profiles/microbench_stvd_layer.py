"""StVD layer discard drawn on the device (csrc/stvd_layer.cu), measured on the GPU:
  (a) selection (vc_stvd_layer_keep) and feature gather kernel time, CUDA events, at n = 14 k, 60 k, 140 k, 215 k rows
      (the stage sizes of BASELINE.md's batches; 215 437 is stage 2 of the 300 k-virtual, uncapped scene);
  (b) graph-replayed training step of VirConvL8x bf16 at bench.py's batch (2 scenes x (16 k LiDAR + 80 k virtual), cap
      40 000 voxels each), discard_mode='spconv2_compat' against 'paper' + discard_rng='device', alternating in one process;
  (c) the same at the 300 k-virtual, uncapped size;
  (d) the module-path paper-mode step (host numpy draws, no executor), for scale.
Prints the device name and power limit with the numbers.

    python profiles/microbench_stvd_layer.py [--steps 40]
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
from virconv_b200 import ops, scenes                                      # noqa: E402
from virconv_b200.backbone import VirConvL8x                              # noqa: E402
from virconv_b200.graph import GraphedStep, masked_mean                   # noqa: E402

CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
DEV = torch.device('cuda:0')


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


def kernels(reps):
    lib = ops._lib.load()
    seed = torch.tensor([7], dtype=torch.int64, device=DEV)
    for n in (14000, 60000, 140000, 215437):
        keep = torch.empty(n, dtype=torch.int32, device=DEV)
        pos = torch.empty(n, dtype=torch.int32, device=DEV)
        kept = torch.empty(1, dtype=torch.int32, device=DEV)
        ws = torch.empty(lib.vc_stvd_layer_keep_ws_bytes(n), dtype=torch.uint8, device=DEV)
        sel = lambda: lib.vc_stvd_layer_keep(None, seed.data_ptr(), 1, n, None, 0.1, keep.data_ptr(), kept.data_ptr(),
                                             pos.data_ptr(), ws.data_ptr(), ws.numel(), ops._stream())
        t_sel = events(sel, reps)
        k = int(kept.item())
        x = torch.randn(n, 32, device=DEV)           # a 16+16-channel concat, the widest discard in VirConv-L is 64
        rows = keep[:k]
        t_g32 = events(lambda: ops.gather_rows(x, rows), reps)
        x64 = torch.randn(n, 64, device=DEV)
        t_g64 = events(lambda: ops.gather_rows(x64, rows), reps)
        print(f'(a) n = {n:7d} -> k = {k:7d}: select {t_sel:7.1f} us | gather fp32 32 ch {t_g32:6.1f} us, 64 ch {t_g64:6.1f} us')


def batch(n_virtual, max_voxels, ids):
    b = scenes.make_batch(ids, 16384, n_virtual, max_voxels, training=True)
    return {'voxel_features': torch.from_numpy(b.voxel_features.copy()).to(DEV),
            'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).to(DEV), 'batch_size': 2, 'calib': b.calib,
            'aug_param': torch.from_numpy(b.aug_param.copy())}


def loss_of(out):
    named = dict(out['multi_scale_3d_features'])
    named['out'] = out['encoded_spconv_tensor']
    return sum(masked_mean(t) for t in named.values())


def graph_steps(label, n_virtual, max_voxels, steps, rounds):
    bs = [batch(n_virtual, max_voxels, [2 * i, 2 * i + 1]) for i in range(2)]
    base = VirConvL8x(CFG, 8, [1408, 1600, 80], precision='bf16')
    fill_module(base, 666)
    base.to(DEV).train()
    arms = {}
    for name, mode, rng in (('off (spconv2_compat)', 'spconv2_compat', 'numpy'), ('on (paper, device)', 'paper', 'device')):
        m = copy.deepcopy(base)
        m.discard_mode, m.discard_rng = mode, rng
        arms[name] = GraphedStep(m, loss_of, margin=1.15)
    times = {k: [] for k in arms}
    for name, g in arms.items():
        for s in range(6):
            g(bs[s % 2])
    torch.cuda.synchronize()
    for _ in range(rounds):                          # alternate the arms
        for name, g in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for s in range(steps):
                g(bs[s % 2])
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3 / steps)
    n0 = bs[0]['voxel_features'].shape[0]
    for name, t in times.items():
        print(f'({label}) {n0} input voxels, StVD layer discard {name}: '
              f'{min(t):.3f} ms/step (min of {rounds} rounds of {steps} replays; all: {", ".join(f"{v:.3f}" for v in t)}); '
              f're-captures {arms[name].recaptures}')


def module_path(steps):
    b = batch(80000, 40000, [0, 1])
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], precision='bf16', discard_mode='paper')
    fill_module(m, 666)
    m.to(DEV).train()

    def one():
        for p in m.parameters():
            p.grad = None
        loss_of(m(dict(b))).backward()
    for _ in range(3):
        one()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        one()
    torch.cuda.synchronize()
    print(f'(d) module path, paper mode, numpy draws, bf16: {(time.perf_counter() - t0) * 1e3 / steps:.3f} ms/step')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--reps', type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    print('device:', card())
    kernels(args.reps)
    graph_steps('b', 80000, 40000, args.steps, args.rounds)
    graph_steps('c', 300000, 10 ** 6, max(args.steps // 4, 5), args.rounds)
    module_path(max(args.steps // 4, 5))
    print('device:', card())


if __name__ == '__main__':
    main()
