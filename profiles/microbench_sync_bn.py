"""SyncBatchNorm on the fast path (sync_bn, vc_exec_forward_sync), measured on the GPU — VirConv-L bf16 training step at
bench.py's batch (2 scenes x (16 k LiDAR + 80 k virtual), cap 40 000 voxels each):
  (a) GraphedStep with BatchNorm1d against the SyncBatchNorm-converted model at world size 1 (same kernels: expected equal);
  (b) GraphedStep of the converted model with a no-op `bn_reducer`: the split conv -> exchange -> BN apply path a multi-rank
      step runs, without any communication (what giving up the fused conv + BN launch costs);
  (c) the eager step of the converted model on the per-operator module path (where tools/train.py --sync_bn used to land)
      against the same eager step through the plan executor;
  (d) two or more GPUs: NCCL world size 2, GraphedStep with and without SyncBatchNorm (rank 0's step time); on a one-GPU
      machine these are printed as "not measured".
Arms of one section alternate in one process.  Prints the device name and power limit with the numbers.

    python profiles/microbench_sync_bn.py [--steps 40] [--rounds 3]
"""
from __future__ import annotations

import argparse
import copy
import os
import subprocess
import sys
import tempfile
import time
from datetime import timedelta

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.testing import fill_module                                    # noqa: E402
from virconv_b200 import executor, scenes                                 # noqa: E402
from virconv_b200.backbone import VirConvL8x                              # noqa: E402
from virconv_b200.graph import GraphedStep, masked_mean                   # noqa: E402

CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])


def card(dev):
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'nvidia-smi unavailable'
    return f'{torch.cuda.get_device_name(dev)} | {q}'


def batch(ids, dev):
    b = scenes.make_batch(ids, 16384, 80000, 40000, training=True)
    return {'voxel_features': torch.from_numpy(b.voxel_features.copy()).to(dev),
            'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).to(dev), 'batch_size': len(ids), 'calib': b.calib,
            'aug_param': torch.from_numpy(b.aug_param.copy())}


def loss_of(out):
    named = dict(out['multi_scale_3d_features'])
    named['out'] = out['encoded_spconv_tensor']
    return sum(masked_mean(t) for t in named.values())


def model(dev):
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], precision='bf16')
    fill_module(m, 666)
    return m.to(dev).train()


def alternate(arms, batches, steps, rounds):
    """{name: fn(batch)} -> {name: [ms per step of each round]}; every arm warmed up first, then rounds alternate."""
    for fn in arms.values():
        for s in range(6):
            fn(batches[s % len(batches)])
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for s in range(steps):
                fn(batches[s % len(batches)])
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3 / steps)
    return times


def report(label, times, steps):
    for name, t in times.items():
        print(f'({label}) {name}: {min(t):.3f} ms/step (min of {len(t)} rounds of {steps} steps; all: '
              f'{", ".join(f"{v:.3f}" for v in t)})', flush=True)


def eager_step(m):
    def one(b):
        for p in m.parameters():
            p.grad = None
        loss_of(m(dict(b))).backward()
    return one


def module_path(fn):
    def one(b):
        executor.ENABLED = False
        try:
            fn(b)
        finally:
            executor.ENABLED = True
    return one


def one_gpu(steps, rounds):
    dev = torch.device('cuda:0')
    bs = [batch([2 * i, 2 * i + 1], dev) for i in range(2)]
    base = model(dev)
    sync = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(base))
    split = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(base))
    split.bn_reducer = lambda slot, key: None
    g = {'BatchNorm1d': GraphedStep(base, loss_of, margin=1.15), 'SyncBatchNorm, world size 1': GraphedStep(sync, loss_of, margin=1.15),
         'SyncBatchNorm, split path (no-op reducer)': GraphedStep(split, loss_of, margin=1.15)}
    times = alternate({k: (lambda b, s=s: s(b)) for k, s in g.items()}, bs, steps, rounds)
    report('a/b GraphedStep', times, steps)
    eager = copy.deepcopy(sync)
    times = alternate({'SyncBatchNorm eager, module path': module_path(eager_step(eager)),
                       'SyncBatchNorm eager, plan executor': eager_step(eager)}, bs, max(steps // 4, 5), rounds)
    report('c eager', times, max(steps // 4, 5))


def worker(rank, init, steps, rounds, out):
    import torch.distributed as dist
    dev = torch.device('cuda:%d' % rank)
    torch.cuda.set_device(dev)
    dist.init_process_group('nccl', init_method=init, rank=rank, world_size=2, timeout=timedelta(seconds=600))
    try:
        bs = [batch([2 * i + rank], dev) for i in range(2)]        # one scene per rank, bench.py's pair split over two
        base = model(dev)
        sync = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(base))
        g = {'BatchNorm1d': GraphedStep(base, loss_of, margin=1.15), 'SyncBatchNorm': GraphedStep(sync, loss_of, margin=1.15)}
        times = alternate({k: (lambda b, s=s: s(b)) for k, s in g.items()}, bs, steps, rounds)
        dist.barrier()
        if rank == 0:
            with open(out, 'w') as f:
                for name, t in times.items():
                    f.write(f'(d) NCCL world size 2, GraphedStep {name}: {min(t):.3f} ms/step (rank 0, min of {len(t)} rounds of '
                            f'{steps} steps; all: {", ".join(f"{v:.3f}" for v in t)})\n')
    finally:
        dist.destroy_process_group()


def two_gpus(steps, rounds):
    if torch.cuda.device_count() < 2:
        print('(d) NCCL world size 2, GraphedStep with and without SyncBatchNorm: not measured (one GPU)')
        return
    with tempfile.TemporaryDirectory() as tmp:
        init, out = 'file://' + os.path.join(tmp, 'rdv'), os.path.join(tmp, 'out.txt')
        procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), '--worker', str(r), init, out, '--steps', str(steps),
                                   '--rounds', str(rounds)]) for r in range(2)]
        try:
            for p in procs:
                p.wait(timeout=1800)
        finally:
            for p in procs:
                if p.poll() is None:
                    p.kill()
                    p.wait()
        print(open(out).read() if os.path.exists(out) else '(d) NCCL world size 2: the ranks failed, not measured', end='')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--worker', nargs=3, default=None, metavar=('RANK', 'INIT', 'OUT'))
    a = ap.parse_args()
    if a.worker:
        worker(int(a.worker[0]), a.worker[1], a.steps, a.rounds, a.worker[2])
        return
    print('device:', card(torch.device('cuda:0')), flush=True)
    one_gpu(a.steps, a.rounds)
    two_gpus(a.steps, a.rounds)


if __name__ == '__main__':
    main()
