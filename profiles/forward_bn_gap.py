"""What BatchNorm costs the forward's critical path in bench.py's graph step: per forward layer, the conv
kernel's duration, the gap from its end to the BN apply's start, the BN apply's duration and the gap to the next conv, from
torch.profiler over ~20 replays of the captured VirConv-L training step (GraphedStep with the in-graph voxeliser, bench's
batch and loss).  With the BN apply fused into the conv (VIRCONV_CONV_BN_FUSED=1) the apply columns read 0 and the conv
column includes it.  Per replay it also prints the index phase: the span from the first index kernel (hash insert, probes,
bitmap lookups, strided-conv count / emit / tables, projections) to the last, the time from the voxeliser's last kernel to the first conv,
and the span of the forward's conv chain.  Run on the GPU:

    python profiles/forward_bn_gap.py [--replays 20]

Prints the card name and power limit with the numbers: a kernel time is only meaningful with what it was measured on."""
import argparse
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
from profiles.graph_step_anatomy import card  # noqa: E402
from virconv_b200 import scenes  # noqa: E402
from virconv_b200.backbone import VirConvL8x  # noqa: E402
from virconv_b200.graph import GraphedStep, masked_mean  # noqa: E402

CONV, APPLY, REDUCE = 'tc_conv_persist', 'bn_apply_relu', 'bn_sums_reduce'
INDEX = re.compile(r'\b(hash_insert|subm_probe|subm_lookup|conv_mark|scan_local|scan_blocks|conv_emit_indices|conv_tables|conv_fwd_lookup|index2uv|g2_[a-z_]+|'
                   r'stvd_gather_idx)_kernel')
VOX = re.compile(r'\b(vox_[a-z]+|vscan_local)_kernel')


def forward_windows(events):
    """events: (start_ns, end_ns, name, stream) of every kernel, all replays -> one list of (sorted) kernel events per
    replay, from its voxeliser's first kernel to its first backward kernel."""
    replays, fwd = [], False
    for ev in sorted(events):
        name = ev[2]
        if 'vox_insert' in name and not fwd:      # (the in-graph voxeliser's first kernel)
            fwd = True
            replays.append([ev])
        elif 'masked_mean_bwd' in name or 'bn_bwd' in name:
            fwd = False
        elif fwd:
            replays[-1].append(ev)
    return replays


def index_phase(events):
    """-> per replay {'idx_span', 'vox_to_conv', 'conv_chain', 'kernels'}: first index kernel start -> last index kernel
    end, voxeliser's last kernel end -> first conv start, first conv start -> last conv end (ns), and per index kernel name
    [launches, summed duration in ns]."""
    out = []
    for evs in forward_windows(events):
        idx = [ev for ev in evs if INDEX.search(ev[2])]
        vox = [ev for ev in evs if VOX.search(ev[2])]
        conv = [ev for ev in evs if CONV in ev[2]]
        if not (idx and vox and conv):
            continue
        kernels = {}
        for ev in idx:
            k = kernels.setdefault(INDEX.search(ev[2]).group(1), [0, 0])
            k[0] += 1
            k[1] += ev[1] - ev[0]
        out.append({'idx_span': max(e[1] for e in idx) - min(e[0] for e in idx),
                    'vox_to_conv': conv[0][0] - max(e[1] for e in vox),
                    'conv_chain': max(e[1] for e in conv) - conv[0][0], 'kernels': kernels})
    return out


def forward_layers(events):
    """events: (start_ns, end_ns, name, stream) of every kernel, all replays.  A replay's forward runs from its voxeliser to
    its first backward kernel (the loss of an early output may run before the forward ends: a graph orders by dependency).
    The forward's layers are a strict chain of conv -> BN kernels; a graph replay may put them on any of its streams, so
    they are ordered by time alone.  Returns one list of layer rows per replay."""
    out = []
    for evs in forward_windows(events):
        chain = [ev for ev in evs if CONV in ev[2] or APPLY in ev[2] or REDUCE in ev[2]]
        layers = []
        for j, ev in enumerate(chain):
            if CONV not in ev[2]:
                continue
            row = {'conv': ev[1] - ev[0], 'gap_apply': 0, 'apply': 0, 'end': ev[1]}
            for nx in chain[j + 1:]:
                if REDUCE in nx[2] or APPLY in nx[2]:
                    if APPLY in nx[2]:
                        row['gap_apply'] = nx[0] - row['end'] + row['gap_apply']
                        row['apply'] = nx[1] - nx[0]
                    else:       # (deterministic mode: the partial-sum reduction sits between conv and apply)
                        row['gap_apply'] += nx[1] - row['end']
                    row['end'] = nx[1]
                else:
                    break
            layers.append(row)
        for a, b in zip(layers, layers[1:]):
            a['gap_next'] = max(0, next(ev[0] for ev in chain if CONV in ev[2] and ev[0] >= a['end']) - a['end'])
        if layers:
            layers[-1]['gap_next'] = 0
        out.append(layers)
    return out


def profile_events(step, batches, replays):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(replays):
            step(batches[i % bench.POOL])
        torch.cuda.synchronize()
    return [(e.start_ns(), e.end_ns(), e.name(), e.device_resource_id()) for e in prof.profiler.kineto_results.events()
            if e.device_type() == torch.autograd.DeviceType.CUDA and e.duration_ns() > 0]


def report(events):
    reps = forward_layers(events)
    n_layers = max(len(r) for r in reps)
    reps = [r for r in reps if len(r) == n_layers]
    R = len(reps)
    print(f'VIRCONV_CONV_BN_FUSED={os.environ.get("VIRCONV_CONV_BN_FUSED", "1")}: {R} replays, {n_layers} forward layers '
          f'(us, mean over replays)')
    print(f'{"layer":>5} {"conv":>8} {"gap->bn":>8} {"bn apply":>9} {"gap->next":>10}')
    cols = ('conv', 'gap_apply', 'apply', 'gap_next')
    tot = dict.fromkeys(cols, 0.0)
    for k in range(n_layers):
        v = {c: sum(r[k][c] for r in reps) / R / 1e3 for c in cols}
        for c in cols:
            tot[c] += v[c]
        print(f'{k:5d} {v["conv"]:8.1f} {v["gap_apply"]:8.1f} {v["apply"]:9.1f} {v["gap_next"]:10.1f}')
    print(f'  sum {tot["conv"]:8.1f} {tot["gap_apply"]:8.1f} {tot["apply"]:9.1f} {tot["gap_next"]:10.1f}')
    print(f'BN apply + both gaps: {(tot["gap_apply"] + tot["apply"] + tot["gap_next"]) / 1e3:.3f} ms/step; '
          f'conv + apply + gaps: {sum(tot.values()) / 1e3:.3f} ms/step')
    ph = index_phase(events)
    print(f'index phase ({len(ph)} replays, us: mean [min, max]):')
    for k, label in (('idx_span', 'first -> last index kernel'), ('vox_to_conv', 'voxeliser end -> first conv'),
                     ('conv_chain', 'first conv start -> last conv end')):
        v = [r[k] / 1e3 for r in ph]
        print(f'  {label:34s} {sum(v) / len(v):8.1f} [{min(v):.1f}, {max(v):.1f}]')
    names = sorted({n for r in ph for n in r['kernels']}, key=lambda n: -sum(r['kernels'].get(n, [0, 0])[1] for r in ph))
    print('  index kernels (per replay: launches, summed duration us; the two index streams overlap):')
    for n in names:
        c = sum(r['kernels'].get(n, [0, 0])[0] for r in ph) / len(ph)
        t = sum(r['kernels'].get(n, [0, 0])[1] for r in ph) / len(ph) / 1e3
        print(f'    {n:20s} {c:6.1f} {t:8.1f}')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--replays', type=int, default=20)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
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
    events = profile_events(step, batches, args.replays)
    print(f'card: {card()}')
    report(events)


if __name__ == '__main__':
    main()
