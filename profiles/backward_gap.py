"""Where the backward of bench.py's graph step waits: per backward layer in walk order, the BatchNorm backward, the input
gradient (dgrad) and the weight gradient (wgrad) kernels, from torch.profiler over ~20 replays of the captured VirConv-L
training step (GraphedStep with the in-graph voxeliser, bench's batch and loss).  The plan executor runs each layer's wgrad
on its own stream beside the main stream's BN backward -> dgrad chain; a cooperative BN grid or a dgrad only starts once
its CTAs fit, so a wgrad launch that fills the SMs delays the main stream.  Columns (us, mean over replays):

  bn / dgrad / wgrad   span of the kernel and its start delay (BN: after the previous main-stream kernel ended; dgrad: after
                       its BN backward; wgrad: after both its BN backward and the previous wgrad ended).  The dgrad column
                       adds up the layer's input-gradient kernels
  passes, ctas         the wgrad launch's grid: blockIdx.y passes, CTAs over all passes
  gap                  main stream idle from this layer's dgrad end to the next layer's BN backward start
  idle|w               time the main stream runs no kernel while a wgrad kernel runs, from this layer's BN backward start
                       to the next one's

Per replay: the backward span (first backward kernel to wgrad_finalize_kernel) and the wgrad tail after the last dgrad.
Run on the GPU:

    python profiles/backward_gap.py [--replays 20] [--wgrad-ctas N]

Prints the card name and power limit with the numbers: a kernel time is only meaningful with what it was measured on."""
import argparse
import json
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
from profiles.graph_step_anatomy import card  # noqa: E402
from virconv_b200 import _lib, scenes  # noqa: E402
from virconv_b200.backbone import VirConvL8x  # noqa: E402
from virconv_b200.graph import GraphedStep, masked_mean  # noqa: E402

BN, WGRAD, FIN = 'bn_bwd', 'tc_wgrad_half_kernel', 'wgrad_finalize_kernel'
DGRAD = re.compile(r'tc_conv_persist_kernel|tc_scatter_kernel|scatter_gemm_kernel|gather_gemm_kernel')
START = re.compile(r'masked_mean_bwd|bn_bwd')


def backward_windows(events):
    """events: (start_us, end_us, name, grid) of every kernel / memset, all replays -> one time-sorted list per replay, from
    its first backward kernel to its wgrad_finalize_kernel."""
    reps, cur = [], None
    for ev in sorted(events):
        if cur is None and START.search(ev[2]):
            cur = []
        if cur is not None:
            cur.append(ev)
            if FIN in ev[2]:
                reps.append(cur)
                cur = None
    return reps


def _busy(intervals, lo, hi):
    """union of the intervals clipped to [lo, hi) -> sorted disjoint list"""
    out = []
    for a, b in sorted((max(a, lo), min(b, hi)) for a, b in intervals if b > lo and a < hi):
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def _overlap(xs, ys):
    t, i, j = 0.0, 0, 0
    while i < len(xs) and j < len(ys):
        a, b = max(xs[i][0], ys[j][0]), min(xs[i][1], ys[j][1])
        t += max(0.0, b - a)
        if xs[i][1] < ys[j][1]:
            i += 1
        else:
            j += 1
    return t


def replay_layers(evs):
    """-> (layer rows in walk order, replay totals) of one replay's backward"""
    bns = [e for e in evs if BN in e[2]]
    wgs = [e for e in evs if WGRAD in e[2]]
    dgs = [e for e in evs if DGRAD.search(e[2])]
    main = [e for e in evs if WGRAD not in e[2] and FIN not in e[2]]
    t0, t_end = evs[0][0], evs[-1][1]
    rows, used, w_prev = [], set(), None
    for i, b in enumerate(bns):
        nxt = bns[i + 1][0] if i + 1 < len(bns) else t_end
        prev_main = max((e[1] for e in main if e[1] <= b[0] and e is not b), default=b[0])
        w = next((e for e in wgs if e[0] >= b[1] - 1e-3 and id(e) not in used), None)
        ds = [e for e in dgs if b[1] - 1e-3 <= e[0] < nxt]      # (a 2-D layer's input gradient may be two kernels)
        row = {'bn': b[1] - b[0], 'bn_delay': b[0] - prev_main}
        if w is not None:
            used.add(id(w))
            ready = max(b[1], w_prev[1]) if w_prev is not None else b[1]
            g = w[3] or (0, 0, 0)
            m = re.search(r'<(\d+), *(\d+)>', w[2])
            row.update(wgrad=w[1] - w[0], wgrad_delay=max(0.0, w[0] - ready), passes=g[1], ctas=g[0] * g[1],
                       shape=f'{m.group(1)}->{m.group(2)}' if m else '?')
            w_prev = w
        if ds:
            row.update(dgrad=sum(e[1] - e[0] for e in ds), dgrad_delay=ds[0][0] - b[1],
                       gap=max(0.0, nxt - ds[-1][1]) if i + 1 < len(bns) else 0.0)
        mb = _busy([(e[0], e[1]) for e in main], b[0], nxt)
        wb = _busy([(e[0], e[1]) for e in wgs], b[0], nxt)
        row['idle_w'] = sum(y - x for x, y in wb) - _overlap(mb, wb)
        rows.append(row)
    last_d = max((e[1] for e in dgs), default=t0)
    fin = next(e for e in evs if FIN in e[2])
    return rows, {'span': fin[1] - t0, 'tail': fin[1] - last_d}


def trace_events(path):
    with open(path) as f:
        tr = json.load(f)
    out = []
    for e in tr.get('traceEvents', []):
        if e.get('ph') == 'X' and e.get('cat') in ('kernel', 'gpu_memset') and e.get('dur', 0) > 0:
            grid = tuple(e.get('args', {}).get('grid', ())) or None
            out.append((float(e['ts']), float(e['ts']) + float(e['dur']), e['name'], grid))
    return out


def report(events):
    reps = [replay_layers(r) for r in backward_windows(events)]
    n = max(len(r[0]) for r in reps)
    reps = [r for r in reps if len(r[0]) == n]
    R = len(reps)
    print(f'{R} replays, {n} backward layers in walk order (us, mean over replays)')
    cols = ('bn', 'bn_delay', 'dgrad', 'dgrad_delay', 'wgrad', 'wgrad_delay', 'gap', 'idle_w')
    print(f'{"layer":>5} {"wgrad":>6} {"passes":>6} {"ctas":>5} {"bn":>7} {"bn dly":>7} {"dgrad":>7} {"dg dly":>7} '
          f'{"wgrad":>7} {"wg dly":>7} {"gap":>7} {"idle|w":>7}')
    tot = dict.fromkeys(cols, 0.0)
    for k in range(n):
        v = {c: sum(r[0][k].get(c, 0.0) for r in reps) / R for c in cols}
        for c in cols:
            tot[c] += v[c]
        r0 = max((r[0][k] for r in reps), key=lambda x: sum(y[0][k].get('shape') == x.get('shape') for y in reps))
        print(f'{k:5d} {r0.get("shape", "-"):>6} {r0.get("passes", 0):6d} {r0.get("ctas", 0):5d} ' +
              ' '.join(f'{v[c]:7.1f}' for c in cols))
    print(f'{"sum":>24} ' + ' '.join(f'{tot[c]:7.1f}' for c in cols))
    for key, label in (('span', 'backward span (first backward kernel -> wgrad_finalize end)'),
                       ('tail', 'wgrad tail (last dgrad end -> wgrad_finalize end)')):
        v = [r[1][key] for r in reps]
        print(f'{label}: {sum(v) / R:.1f} us [{min(v):.1f}, {max(v):.1f}]')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--replays', type=int, default=20)
    ap.add_argument('--time-replays', type=int, default=50, help='replays timed with CUDA events before profiling')
    ap.add_argument('--wgrad-ctas', type=int, default=0, help='CTA cap of each wgrad launch (0: the executor default)')
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    lib = _lib.load()
    _lib.check(lib.vc_conv_wgrad_tc3_config(1, args.wgrad_ctas), 'vc_conv_wgrad_tc3_config')
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

    torch.manual_seed(666)
    model = VirConvL8x(bench.CFG, 8, [1408, 1600, 80], precision='bf16').to(dev).train()
    step = GraphedStep(model, loss_of, list(model.parameters()), margin=float(os.environ.get('VIRCONV_GRAPH_MARGIN', '1.15')),
                       voxelizer=vox)
    for i in range(3 * bench.POOL):
        step(batches[i % bench.POOL])
    torch.cuda.synchronize()
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(args.time_replays):
        step(batches[i % bench.POOL])
    e.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(e) / max(args.time_replays, 1)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.replays):
            step(batches[i % bench.POOL])
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'trace.json')
        prof.export_chrome_trace(path)
        events = trace_events(path)
    print(f'card: {card()}')
    print(f'wgrad CTA cap {args.wgrad_ctas or "default"}; {args.time_replays} replays without the profiler: '
          f'{ms:.3f} ms/step')
    report(events)


if __name__ == '__main__':
    main()
