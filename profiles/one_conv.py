"""Run ONE conv layer of the bench workload a few times (for ncu captures of a single launch).
    LAYER=6 REPS=4 python profiles/one_conv.py       # layer index as printed by microbench_conv2.py"""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from virconv_b200 import _lib, executor, ops, scenes
from virconv_b200.backbone import VirConvL8x

dev = torch.device('cuda:0')
lib = _lib.load()
_lib.check(lib.vc_conv_tc2_config(int(os.environ.get('VIRCONV_TC2_CTAS', '0'))), 'vc_conv_tc2_config')
torch.manual_seed(666)
model = VirConvL8x(bench.CFG, 8, [1408, 1600, 80], precision='bf16').to(dev).train()
executor.ENABLED = False
b = scenes.make_batch([0, 1], training=True)
calls = []
orig = ops.conv_forward


def spy(feats, weight, rb, bn_sums=None, precision='fp32', feats_bf16=None, keep=None):
    calls.append((feats.detach(), weight.detach(), rb))
    return orig(feats, weight, rb, bn_sums, precision, feats_bf16, keep)


ops.conv_forward = spy
with torch.no_grad():
    model({'voxel_features': torch.from_numpy(b.voxel_features).to(dev), 'voxel_coords': torch.from_numpy(b.voxel_coords).to(dev),
           'batch_size': 2, 'calib': b.calib, 'aug_param': b.aug_param})
ops.conv_forward = orig
li = int(os.environ.get('LAYER', '6'))
feats, weight, rb = calls[li]
cout, cin = weight.shape[0], weight.shape[-1]
fb = ops.cast_bf16(feats.contiguous())
ws = ops._ws(lib.vc_conv_tc_ws_bytes(cin, cout, rb.K), dev)
out = torch.empty((rb.n_out, cout), dtype=torch.float32, device=dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
torch.cuda.synchronize()
for _ in range(int(os.environ.get('REPS', '4'))):
    flush.zero_()
    _lib.check(lib.vc_conv_fwd_tc(ops._p(fb), ops._p(weight.contiguous()), ops._p(rb.nbr), ops._p(out), rb.n_out, cin, cout, rb.K,
                                  None, ops._p(ws), ws.numel(), ops._p(ops.tc_error_flag(dev)), ops._stream()), 'fwd')
torch.cuda.synchronize()
print('layer', li, cin, cout, rb.K, rb.n_out, 'err', int(ops.tc_error_flag(dev).item()))
