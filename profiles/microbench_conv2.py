"""The tensor-core conv kernel on the bench workload, per layer.
    python profiles/microbench_conv2.py            # VIRCONV_LIB=<.so> times another build of the library
For every conv layer of VirConv-L on the bench batch: forward and gather-dgrad through the C ABI (weight-image prep
launch included in both), median of 7 CUDA-event timings with the L2 flushed in between, and the maximum relative
difference to the fp32 kernel fed bf16-rounded operands.  Each layer line ends with the kernel's shared-memory plan
(vc_conv_tc2_plan: ring stages S, resident weights w or streamed s, CTAs per SM) for the forward timed here, the forward
with BatchNorm sums of the training step (fwd+bn) and the dgrad."""
import ctypes
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from virconv_b200 import _lib, ops, scenes
from virconv_b200.backbone import VirConvL8x

dev = torch.device('cuda:0')
lib = _lib.load()
_lib.check(lib.vc_conv_tc2_config(int(os.environ.get('VIRCONV_TC2_CTAS', '0'))), 'vc_conv_tc2_config')
torch.manual_seed(666)
model = VirConvL8x(bench.CFG, 8, [1408, 1600, 80], precision='bf16').to(dev).train()
os.environ['VIRCONV_EXECUTOR'] = '0'
from virconv_b200 import executor
executor.ENABLED = False          # module path: ops.conv_forward is called per layer
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


def plan(kc, nr, K, bn_sums=0):
    out = (ctypes.c_int32 * 4)()
    _lib.check(lib.vc_conv_tc2_plan(kc, nr, K, bn_sums, out), 'vc_conv_tc2_plan')
    return f'S={out[0]}{"w" if out[1] else "s"}x{out[2]}'


tot = {}
for li, (feats, weight, rb) in enumerate(calls):
    cout, cin = weight.shape[0], weight.shape[-1]
    feats = feats.contiguous()
    weight = weight.contiguous()
    fb = ops.cast_bf16(feats)
    dout = torch.randn(rb.n_out, cout, device=dev)
    db = ops.cast_bf16(dout)
    ws = _ws(lib.vc_conv_tc_ws_bytes(cin, cout, rb.K), dev)
    gather_dgrad = not (rb.subm and not rb.unique_coords)
    res = {}

    out = torch.empty((rb.n_out, cout), dtype=torch.float32, device=dev)
    res['fwd'] = timed(lambda: _lib.check(lib.vc_conv_fwd_tc(_p(fb), _p(weight), _p(rb.nbr), _p(out), rb.n_out, cin, cout, rb.K,
                                                             None, _p(ws), ws.numel(), _p(err), _stream()), 'vc_conv_fwd_tc'))
    d_f = rel(out, ops.conv_forward(bf16r(feats), bf16r(weight), rb, None, 'fp32'))
    d_d = None
    if gather_dgrad:
        din = torch.empty((rb.n_in, cin), dtype=torch.float32, device=dev)
        table, mirror = (rb.nbr, 1) if rb.subm else (rb.nbr_bwd, 0)
        res['dgrad'] = timed(lambda: _lib.check(lib.vc_conv_dgrad_tc(_p(db), _p(weight), _p(table), _p(din), rb.n_in, cin, cout, rb.K,
                                                                     mirror, _p(ws), ws.numel(), _p(err), _stream()), 'vc_conv_dgrad_tc'))
        d_d = rel(din, ops.conv_dgrad(bf16r(dout), bf16r(weight), rb, 'fp32'))
    for k, v in res.items():
        tot[k] = tot.get(k, 0.0) + v
    P = rb.n_pairs()
    by = feats.shape[0] * cin * 2 + rb.n_out * cout * 4 + P * 8 + rb.K * cin * cout * 2
    print(f'L{li:02d} {"subm" if rb.subm else "conv"}{rb.ndim}d {cin:2d}->{cout:2d} K={rb.K:2d} N_in={feats.shape[0]:6d} N_out={rb.n_out:6d} '
          f'P={P:8d} ' + ' '.join(f'{k}={v:6.1f}us' for k, v in sorted(res.items())) +
          f'  fwd: {by / res["fwd"] / 1e3:7.1f} GB/s {2 * P * cin * cout / res["fwd"] / 1e6:6.1f} TF/s'
          f'  maxrel fwd {d_f:.1e}' + (f' dgrad {d_d:.1e}' if d_d is not None else '') +
          f'  plan fwd {plan(cin, cout, rb.K)} fwd+bn {plan(cin, cout, rb.K, 1)}' + (f' dgrad {plan(cout, cin, rb.K)}' if gather_dgrad else ''), flush=True)
print('TOTAL us', {k: round(v, 1) for k, v in sorted(tot.items())})
print('error flag', int(err.item()))
