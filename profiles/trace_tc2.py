"""Pipeline timeline of the persistent wgmma conv kernel (debug build -DVC_TC_TRACE: python -c "from virconv_b200 import
build; build.build(defines=['VC_TC_TRACE'], suffix='trace')", run with VIRCONV_LIB=virconv_b200/lib/libvirconv_sm90_trace.so).
CTA 0's events in ns since kernel start: tables published, stages issued / consumed, tiles committed, epilogue start / end."""
import ctypes
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import bench
from virconv_b200 import _lib, executor, ops, scenes
from virconv_b200.backbone import VirConvL8x

dev = torch.device('cuda:0')
torch.manual_seed(666)
model = VirConvL8x(bench.CFG, 8, [1408, 1600, 80], precision='bf16').to(dev).train()
executor.ENABLED = False
b = scenes.make_batch([0, 1], training=True)
calls = []
orig = ops.conv_forward


def spy(feats, weight, rb, bn_sums=None, precision='fp32', feats_bf16=None, keep=None):
    calls.append((feats.detach(), weight.detach(), rb, precision))
    return orig(feats, weight, rb, bn_sums, precision, feats_bf16, keep)


ops.conv_forward = spy
with torch.no_grad():
    model({'voxel_features': torch.from_numpy(b.voxel_features).to(dev), 'voxel_coords': torch.from_numpy(b.voxel_coords).to(dev),
           'batch_size': 2, 'calib': b.calib, 'aug_param': b.aug_param})
ops.conv_forward = orig
lib = _lib.load()
_lib.check(lib.vc_conv_tc2_config(int(os.environ.get('VIRCONV_TC2_CTAS', '0'))), 'vc_conv_tc2_config')
lib.vc_debug_set_trace2.argtypes = [ctypes.c_void_p]
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
names = ['table published', 'stage issued', 'stage consumed', 'tile committed', 'epilogue start', 'epilogue end', 'misc']
for li in [int(x) for x in os.environ.get('LAYERS', '2,6,10').split(',')]:
    feats, weight, rb, prec = calls[li]
    fb = ops.cast_bf16(feats)
    ops.conv_forward(feats, weight, rb, None, prec, fb)
    for cold in (1, 0):
        trace = torch.zeros(9 * 256, dtype=torch.int64, device=dev)
        if cold:
            flush.zero_()
        assert lib.vc_debug_set_trace2(trace.data_ptr()) == 0
        ops.conv_forward(feats, weight, rb, None, prec, fb)
        torch.cuda.synchronize()
        lib.vc_debug_set_trace2(None)
        t = trace.cpu().numpy().reshape(9, 256)
        t0 = t[6][0]
        print(f'layer {li}: {weight.shape[-1]}->{weight.shape[0]} K={rb.K} N={rb.n_out} {"L2 flushed" if cold else "warm"} (ns since CTA 0 start)')
        for r in range(7):
            v = t[r][t[r] > 0] - t0
            print(f'  {names[r]:16s} n={len(v):3d}: ' + ' '.join(str(int(x)) for x in v[:40]))
        # SM-clock phase stamps inside a stage (cycles since the role's first stamp)
        for r, nph, what in ((7, 4, 'producer leader [top, slot free, copies issued, retired]'), (8, 3, 'MMA thread [before wait, landed, issued]')):
            v = t[r][t[r] > 0]
            if len(v):
                v = v - v[0]
                rows = [' '.join('%6d' % int(x) for x in v[i:i + nph]) for i in range(0, min(len(v), nph * 24), nph)]
                print(f'  cycles, {what}:')
                for row in rows:
                    print('      ' + row)
