"""The parameter update after loss.backward() (train_utils.py:50-52), three questions in one process, arms alternating:
  (a) torch   — the reference's update over torch on the GPU: clip_grad_norm_, one p.mul_ per tensor for the true weight
                decay (fastai_optim.py:136-147), torch.optim.Adam (foreach) with this step's momentum;
  (b) fused   — optim.FusedAdamOneCycle.step(): vc_optim_step, two launches;
      both on the VirConv-T backbone's tensors (VirConv8x, MM) and on a detector-sized set (the same tensors plus synthetic
      ones up to ~13 M elements): host time per call ending in a synchronise, device time from CUDA events, L2 flushed (256
      MiB write) before every call; for the fused arm the achieved bytes/s counted as 32 B per parameter (norm pass: read g;
      update pass: read p, g, m, v, write p, m, v) over the event time, against the H100 SXM data sheet's 3.35 TB/s;
  (c) a VirConv-T bf16 GraphedStep at microbench_graph_t.py's workload followed by (a), followed by (b), and with the update
      inside the graph: time per whole iteration, lr / mom set every iteration as OneCycle does.
Prints the device name and power limit with the numbers, and the largest parameter difference between the arms after the
timed windows.

    python profiles/microbench_optim.py [--steps 40] [--rounds 5]
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
from virconv_b200.optim import FusedAdamOneCycle, leaf_param_groups       # noqa: E402

CFG_T = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.15, NUM_FILTERS=[16, 32, 64, 64], MM=True)
N_LIDAR, N_VIRTUAL, MAX_VOXELS, POOL = 16384, 80000, 16000, 4            # microbench_graph_t.py's workload
MARGIN = 1.15
WD, MAX_NORM = 0.01, 10.0
HBM_PEAK = 3.35e12                                                        # H100 SXM data sheet, bytes/s
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


def schedule(i):
    return 0.001 + 1e-5 * (i % 100), 0.95 - 1e-4 * (i % 100)


class TorchArm:
    """(a): what the reference's loop does with torch on [non-BN, BN] groups."""

    def __init__(self, groups):
        self.groups = groups
        self.params = groups[0] + groups[1]
        self.adam = torch.optim.Adam([{'params': g, 'lr': 0} for g in groups], betas=(0.9, 0.99))
        self.lr, self.mom = 3e-3, 0.9

    def step(self):
        torch.nn.utils.clip_grad_norm_(self.params, MAX_NORM)
        with torch.no_grad():
            for p in self.params:
                p.mul_(1 - WD * self.lr)
        for g in self.adam.param_groups:
            g['lr'], g['betas'] = self.lr, (self.mom, 0.99)
        self.adam.step()


class FusedArm:
    def __init__(self, groups):
        self.params = groups[0] + groups[1]
        self.opt = FusedAdamOneCycle(groups, wd=WD)

    def step(self):
        self.opt.lr, self.opt.mom = self.lr, self.mom
        self.opt.step(max_norm=MAX_NORM)


def param_sets():
    m = VirConv8x(CFG_T, 8, [1408, 1600, 80])
    fill_module(m, 667)
    groups, rest = leaf_param_groups(m.to(DEV))
    assert not rest
    gen = torch.Generator(device='cpu').manual_seed(3)
    big = [torch.nn.Parameter((torch.randn(n, generator=gen) * 0.05).to(DEV))
           for n in (4 << 20, 3 << 20, 2 << 20, 1 << 20, 1 << 20, 600000, 300001)]
    return {'VirConv-T backbone': groups, 'detector-sized': [groups[0] + big, groups[1]]}


def time_arms(arms, steps, rounds, before_step, flush):
    """-> {arm: (device ms per call, host ms per call ending in a synchronise)}, medians of the rounds"""
    dev = {k: [] for k in arms}
    host = {k: [] for k in arms}
    it = 0
    for _ in range(rounds):
        for name, fn in arms.items():
            d, h = [], []
            for _ in range(steps):
                before_step(name, it)
                it += 1
                flush.zero_()
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                a.record()
                fn()
                e.record()
                torch.cuda.synchronize()
                h.append((time.perf_counter() - t0) * 1e3)
                d.append(a.elapsed_time(e))
            dev[name].append(statistics.mean(d))
            host[name].append(statistics.mean(h))
    return {k: (statistics.median(dev[k]), min(dev[k]), max(dev[k]), statistics.median(host[k])) for k in arms}


def bench_update(name, groups, args, flush):
    n = sum(p.numel() for g in groups for p in g)
    tensors = sum(len(g) for g in groups)
    twins = {k: [[torch.nn.Parameter(p.detach().clone()) for p in g] for g in groups] for k in ('torch', 'fused')}
    arms = {'torch': TorchArm(twins['torch']), 'fused': FusedArm(twins['fused'])}
    gen = torch.Generator(device='cpu').manual_seed(11)
    grads = [(torch.randn(p.numel(), generator=gen) * 1e-2).view_as(p).to(DEV) for g in groups for p in g]

    def before(arm, it):
        a = arms[arm]
        a.lr, a.mom = schedule(it)
        for p, g in zip(a.params, grads):
            if p.grad is None:
                p.grad = g.clone()
            else:
                p.grad.copy_(g)             # (torch's clip_grad_norm_ scales the gradients in place: restore them)

    lib = _lib.load()
    for arm in arms:                        # warm-up: every shape once through every arm
        for it in range(3):
            before(arm, it)
            arms[arm].step()
    torch.cuda.synchronize()
    l0 = lib.vc_launch_count()
    before('fused', 0)
    arms['fused'].step()
    launches = lib.vc_launch_count() - l0
    res = time_arms({k: a.step for k, a in arms.items()}, args.steps, args.rounds, before, flush)
    print(f'{name}: {tensors} tensors, {n} parameters')
    for k, (d, lo, hi, h) in res.items():
        extra = ''
        if k == 'fused':
            bps = 32.0 * n / (d * 1e-3)
            extra = (f'; {launches} launches; {bps / 1e9:.0f} GB/s counted as 32 B per parameter over the event time = '
                     f'{100 * bps / HBM_PEAK:.1f} % of the data sheet\'s 3.35 TB/s')
        print(f'  {k:6s} {d:7.3f} ms/call device (median of rounds; min {lo:.3f}, max {hi:.3f}), {h:7.3f} ms/call host, '
              f'synchronised{extra}')
    # the arms ran different numbers of steps from the warm-up on, so compare one more step from a common state
    with torch.no_grad():
        for p, q in zip(arms['torch'].params, arms['fused'].params):
            q.copy_(p)
    sd = arms['torch'].adam.state_dict()
    arms['fused'].opt.load_state_dict(sd)
    for arm in arms:
        before(arm, 7)
        arms[arm].step()
    torch.cuda.synchronize()
    diff = max(float((p.detach() - q.detach()).abs().max()) for p, q in zip(arms['torch'].params, arms['fused'].params))
    print(f'  largest parameter difference between the arms after one more step from the same state: {diff:.3e}')


def bench_iteration(args, flush):
    bs = []
    for i in range(POOL):
        b = scenes.make_batch_mm([2 * i, 2 * i + 1], N_LIDAR, N_VIRTUAL, MAX_VOXELS, training=True)
        bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
        bd.update(batch_size=b.batch_size, calib=b.calib, aug_param=torch.from_numpy(b.aug_param))
        bs.append(bd)
    base = VirConv8x(CFG_T, 8, [1408, 1600, 80], precision='bf16')
    fill_module(base, 667)
    base.to(DEV).train()
    models = {k: copy.deepcopy(base) for k in ('graph + torch', 'graph + fused', 'graph with update')}
    groups = {k: leaf_param_groups(m)[0] for k, m in models.items()}
    torch_arm = TorchArm(groups['graph + torch'])
    opt_e = FusedAdamOneCycle(groups['graph + fused'], wd=WD)
    opt_g = FusedAdamOneCycle(groups['graph with update'], wd=WD)
    g_t = GraphedStep(models['graph + torch'], loss_of, margin=MARGIN)
    g_e = GraphedStep(models['graph + fused'], loss_of, margin=MARGIN)
    g_g = GraphedStep(models['graph with update'], loss_of, margin=MARGIN, optimizer=opt_g, max_grad_norm=MAX_NORM)
    state = {'it': 0}

    def it_torch():
        torch_arm.lr, torch_arm.mom = schedule(state['it'])
        g_t(bs[state['it'] % POOL])
        torch_arm.step()

    def it_fused():
        opt_e.lr, opt_e.mom = schedule(state['it'])
        g_e(bs[state['it'] % POOL])
        opt_e.step(max_norm=MAX_NORM)

    def it_graph():
        opt_g.lr, opt_g.mom = schedule(state['it'])
        g_g(bs[state['it'] % POOL])

    arms = {'graph + torch': it_torch, 'graph + fused': it_fused, 'graph with update': it_graph}

    def before(arm, it):
        state['it'] = it

    for fn in arms.values():                 # captures, allocator pools, every batch through every arm
        for it in range(2 * POOL):
            state['it'] = it
            fn()
    torch.cuda.synchronize()
    # the three arms from one state, the same iterations each: how far apart the parameters end up
    for m in list(models.values())[1:]:
        m.load_state_dict(models['graph + torch'].state_dict())
    opt_e.load_state_dict(torch_arm.adam.state_dict())
    opt_g.load_state_dict(torch_arm.adam.state_dict())
    for it in range(8):
        state['it'] = it
        for fn in arms.values():
            fn()
    torch.cuda.synchronize()
    ref = list(models['graph + torch'].parameters())
    diffs = {k: max(float((p.detach() - q.detach()).abs().max()) for p, q in zip(ref, models[k].parameters()))
             for k in list(models)[1:]}
    res = time_arms(arms, args.steps, args.rounds, before, flush)
    assert int(ops.tc_error_flag(DEV).item()) == 0, 'tensor-core pipeline timeout flag set'
    print(f'VirConv-T bf16 iteration (GraphedStep + update), batch 2, {N_LIDAR} LiDAR + {N_VIRTUAL} virtual points per scene, '
          f'lr / mom set every iteration:')
    for k, (d, lo, hi, h) in res.items():
        print(f'  {k:18s} {d:7.3f} ms/iteration device (median of rounds; min {lo:.3f}, max {hi:.3f}), {h:7.3f} ms host, synchronised')
    print(f'  library launches per replay: {g_e.launches_per_replay} without, {g_g.launches_per_replay} with the update; '
          f'skipped steps {opt_g.skipped_steps()}, re-captures {g_g.recaptures}')
    print('  largest parameter difference from graph + torch after 8 iterations from one state (bf16 step, atomics in the '
          'backward): ' + ', '.join(f'{k} {v:.3e}' for k, v in diffs.items()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    print('device:', card())
    print(f'{args.rounds} rounds x {args.steps} calls per arm, arms alternating, L2 flushed before each call')
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=DEV)
    for name, groups in param_sets().items():
        bench_update(name, groups, args, flush)
    bench_iteration(args, flush)


if __name__ == '__main__':
    main()
