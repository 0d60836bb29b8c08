"""Where the time of bench.py's graph step goes: busy time and launch count per kernel name over ~20 replays of the
captured VirConv-L training step (GraphedStep with the in-graph voxeliser, bench's batch and loss), from torch.profiler
with CUDA activities.  Run on the GPU:

    python profiles/graph_step_anatomy.py [--replays 20] [--top 40]

Prints the card name and power limit with the numbers: a kernel time is only meaningful with what it was measured on."""
import argparse
import os
import re
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
from virconv_b200 import scenes  # noqa: E402
from virconv_b200.backbone import VirConvL8x  # noqa: E402
from virconv_b200.graph import GraphedStep, masked_mean  # noqa: E402

# kernel-name groups the step is summarised by (first match wins)
GROUPS = [('conv fwd / dgrad (tc)', r'tc_conv_persist|tc2_'), ('wgrad (tc)', r'wgrad'), ('scatter dgrad', r'scatter'),
          ('concat', r'cat2'), ('BatchNorm', r'bn_'), ('rulebook / index', r'rulebook|subm|hash|index2uv|count|emit|voxel'),
          ('weight images', r'prep'), ('loss', r'masked_mean'), ('memset / memcpy', r'(?i)^memset|^memcpy'),
          ('torch elementwise / reduce', r'at::|elementwise|reduce_kernel|vectorized|unrolled'), ('other', r'.')]


def card():
    try:
        return subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # (the numbers stay valid; only their label is missing)
        return f'unknown ({e})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--replays', type=int, default=20)
    ap.add_argument('--top', type=int, default=40)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    torch.manual_seed(666)
    model = VirConvL8x(bench.CFG, 8, [1408, 1600, 80], precision='bf16').to(dev).train()
    params = list(model.parameters())
    batches = []
    for i in range(bench.POOL):
        pb = scenes.make_points_batch([2 * i, 2 * i + 1], bench.N_LIDAR, bench.N_VIRTUAL, training=True)
        batches.append({'points': torch.from_numpy(pb.points).to(dev), 'batch_size': pb.batch_size, 'calib': pb.calib,
                        'aug_param': pb.aug_param})
    vox = dict(point_cloud_range=(0, -40, -3, 70.4, 40, 1), voxel_size=(0.05, 0.05, 0.05), max_points_per_voxel=5,
               max_voxels=bench.MAX_VOXELS, vfe_model='max')

    def loss_of(out):
        loss = masked_mean(out['encoded_spconv_tensor'])
        for t in out['multi_scale_3d_features'].values():
            loss = loss + masked_mean(t)
        return loss

    step = GraphedStep(model, loss_of, params, margin=float(os.environ.get('VIRCONV_GRAPH_MARGIN', '1.15')), voxelizer=vox)
    for i in range(3 * bench.POOL):
        step(batches[i % bench.POOL])
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.replays):
            step(batches[i % bench.POOL])
        torch.cuda.synchronize()
    busy = defaultdict(lambda: [0, 0.0])
    for e in prof.profiler.kineto_results.events():
        if e.device_type() == torch.autograd.DeviceType.CUDA and e.duration_ns() > 0:
            b = busy[e.name()]
            b[0] += 1
            b[1] += e.duration_ns() / 1e3
    R = args.replays
    tot_us = sum(v[1] for v in busy.values()) / R
    tot_n = sum(v[0] for v in busy.values()) / R
    print(f'card: {card()}')
    print(f'graph step, {R} replays: device busy {tot_us / 1e3:.3f} ms/step (sum over streams), {tot_n:.0f} device ops/step, '
          f'{step.launches_per_replay} library kernels per replay')
    grp = defaultdict(lambda: [0, 0.0])
    for name, (n, us) in busy.items():
        g = next(g for g, pat in GROUPS if re.search(pat, name))
        grp[g][0] += n
        grp[g][1] += us
    print('by group (us/step, ops/step):')
    for g, (n, us) in sorted(grp.items(), key=lambda kv: -kv[1][1]):
        print(f'  {us / R:9.1f} us  n={n / R:6.1f}  {g}')
    print(f'top {args.top} kernels (us/step, launches/step):')
    for name, (n, us) in sorted(busy.items(), key=lambda kv: -kv[1][1])[:args.top]:
        print(f'  {us / R:9.1f} us  n={n / R:6.1f}  {name[:110]}')


if __name__ == '__main__':
    main()
