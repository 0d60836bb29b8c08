"""The tensor-core weight-gradient kernel on the bench workload, per layer, through the per-operator C ABI.
    python profiles/microbench_wgrad2.py            # VIRCONV_LIB=<.so> times another build of the library
For every conv layer of VirConv-L on the bench batch: median of 7 CUDA-event timings of vc_conv_wgrad_tc (scratch zeroing and
the transposing finalize included) with the L2 flushed in between, and the maximum relative difference to the fp32 kernel
fed bf16-rounded operands."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from virconv_b200 import _lib, executor, ops, scenes
from virconv_b200.backbone import VirConvL8x

dev = torch.device('cuda:0')
lib = _lib.load()
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
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
_p, _ws, _stream = ops._p, ops._ws, ops._stream
err = ops.tc_error_flag(dev)


def timed(fn, reps=7):
    fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(e) * 1e3)
    return sorted(ts)[len(ts) // 2]


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def bf16r(t):
    return t.to(torch.bfloat16).to(torch.float32)


tot = 0.0
for li, (feats, weight, rb) in enumerate(calls):
    cout, cin = weight.shape[0], weight.shape[-1]
    feats = feats.contiguous()
    fb = ops.cast_bf16(feats)
    dout = torch.randn(rb.n_out, cout, device=dev)
    db = ops.cast_bf16(dout)
    ws = _ws(lib.vc_conv_wgrad_tc_ws_bytes(rb.n_out, cin, cout, rb.K), dev)
    dw = torch.empty(tuple(weight.shape), dtype=torch.float32, device=dev)
    t = timed(lambda: _lib.check(lib.vc_conv_wgrad_tc(_p(fb), _p(db), _p(rb.nbr), _p(dw), rb.n_out, cin, cout, rb.K, _p(ws),
                                                      ws.numel(), _p(err), _stream()), 'vc_conv_wgrad_tc'))
    d = rel(dw, ops.conv_wgrad(bf16r(feats), bf16r(dout), weight.shape, rb, 'fp32'))
    tot += t
    P = rb.n_pairs()
    by = (feats.shape[0] * cin + rb.n_out * cout) * 2 + P * 8 + rb.K * cin * cout * 4
    print(f'L{li:02d} {"subm" if rb.subm else "conv"}{rb.ndim}d {cin:2d}->{cout:2d} K={rb.K:2d} N_out={rb.n_out:6d} P={P:8d} '
          f'wgrad={t:6.1f}us  {by / t / 1e3:7.1f} GB/s {2 * P * cin * cout / t / 1e6:6.1f} TF/s  maxrel {d:.1e}', flush=True)
print('TOTAL us', round(tot, 1))
print('error flag', int(err.item()))
