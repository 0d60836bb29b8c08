"""Operators of the VirConv sparse-conv hot path: thin PyTorch wrappers over the C ABI
(include/virconv_b200.h).  PyTorch supplies device memory, streams and autograd plumbing only; every
number is produced by the sm_90a kernels in virconv_b200/csrc.  CUDA tensors are mandatory — there is
no CPU path.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _lib
from ._lib import check, host_f32, host_i32

TILE_ROWS = 128


def _require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise _lib.VirConvLibraryError(
                'virconv_b200 operators run on CUDA tensors only (sm_90a kernels); got a %s tensor. '
                'There is no CPU fallback.' % t.device)


def _stream():
    # raw cudaStream_t of torch's current stream (torch.cuda.current_stream() costs ~10 us per call)
    return torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice())


def _p(t):
    return None if t is None else t.data_ptr()


def _tup(v, nd):
    if isinstance(v, (list, tuple)):
        assert len(v) == nd, (v, nd)
        return tuple(int(x) for x in v)
    return (int(v),) * nd


_WS = {}


def _ws(nbytes, device):
    """Scratch for one C-ABI call.  One persistent, geometrically grown buffer per device: every user is a kernel
    sequence enqueued on the current stream by a single call (or the count/fill pair of the strided rulebook, which
    has no other call in between), so stream order makes reuse safe."""
    nbytes = max(int(nbytes), 256)
    key = (device.type, device.index, _stream())      # one scratch buffer per stream (side-stream work has its own)
    buf = _WS.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(nbytes, 2 * (buf.numel() if buf is not None else 0), 1 << 24), dtype=torch.uint8,
                          device=device)
        _WS[key] = buf
    return buf


# ------------------------------------------------------------------------------------------------
# side stream: the voxel->pixel projection + the 2-D rulebook of an NRConv block run next to its two 3-D convs instead of
# serialising behind those latency-bound kernels.  Joined back into the main stream before anything consumes the
# results; disable with VIRCONV_OVERLAP=0.
# ------------------------------------------------------------------------------------------------
import os as _os

OVERLAP = _os.environ.get('VIRCONV_OVERLAP', '1') != '0'
_SIDE = {}


class _Side:
    def __init__(self, device):
        # high priority: the side stream carries the small index kernels the HOST waits on (row counts of the strided
        # convs); they must not queue behind the wide feature kernels of the main stream
        self.stream = torch.cuda.Stream(device=device, priority=-1)


def side(device) -> _Side:
    key = (device.type, device.index)
    if key not in _SIDE:
        _SIDE[key] = _Side(device)
    return _SIDE[key]


_SIDE2 = {}


def side2(device):
    """Second index stream of the plan executor (image-branch projection + 2-D rulebooks)."""
    key = (device.type, device.index)
    if key not in _SIDE2:
        _SIDE2[key] = torch.cuda.Stream(device=device)
    return _SIDE2[key]


def _keep_alive_on(stream, *tensors):
    for t in tensors:
        if t is not None:
            t.record_stream(stream)


class StatsArena:
    """Zeroed float64 scratch for the BatchNorm channel sums (forward [2,C] + backward [2,C] per layer).  One buffer
    per device; `reset()` (called once per backbone forward) re-zeroes it with a single memset and rewinds the cursor;
    each conv+BN layer takes a fresh slice, so no per-layer memset is needed.  Past the end (or without a reset
    between uses) it falls back to a fresh zeros tensor."""
    SIZE = 16384   # doubles: 64 layers x 4 x 64 channels

    def __init__(self, device):
        self.buf = torch.zeros(self.SIZE, dtype=torch.float64, device=device)
        self.cursor = 0
        self.dirty = False
        self.generation = 0

    def reset(self):
        if self.dirty:
            self.buf.zero_()
        self.cursor = 0
        self.dirty = False
        self.generation += 1

    def take(self, n):
        if self.cursor + n > self.SIZE:
            return torch.zeros(n, dtype=torch.float64, device=self.buf.device)
        out = self.buf[self.cursor:self.cursor + n]
        self.cursor += n
        self.dirty = True
        return out


_ARENAS = {}


def stats_arena(device) -> StatsArena:
    key = (device.type, device.index)
    if key not in _ARENAS:
        _ARENAS[key] = StatsArena(device)
    return _ARENAS[key]


class KernelTimer:
    """Optional per-call CUDA-event timing of the C-ABI calls (bench.py's roofline pass).  Off by default:
    `ops.TIMER = KernelTimer()` turns it on, `ops.TIMER = None` off.  Events are recorded on the launching
    stream; `summary()` synchronises once and returns {name: (calls, total_ms, alg_bytes, flops)}."""

    def __init__(self):
        self.records = []

    def run(self, name, alg_bytes, flops, fn):
        a = torch.cuda.Event(enable_timing=True)
        b = torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        self.records.append((name, a, b, alg_bytes, flops))
        return out

    def summary(self):
        torch.cuda.synchronize()
        agg = {}
        for name, a, b, by, fl in self.records:
            c = agg.setdefault(name, [0, 0.0, 0, 0])
            c[0] += 1
            c[1] += a.elapsed_time(b)
            c[2] += by() if callable(by) else by
            c[3] += fl() if callable(fl) else fl
        return {k: tuple(v) for k, v in agg.items()}


TIMER = None


def _timed(name, alg_bytes, flops, fn):
    if TIMER is None:
        return fn()
    return TIMER.run(name, alg_bytes, flops, fn)


# ------------------------------------------------------------------------------------------------
# precision: 'fp32' = CUDA-core fp32 kernels (1e-4 parity path); 'bf16' = wgmma tensor-core kernels for the
# gathered contractions (bf16 operands, fp32 accumulation in registers, fp32 outputs) where the channel counts allow
# ------------------------------------------------------------------------------------------------
_TC_ERR = {}


def tc_error_flag(device):
    """Persistent device int32 the tensor-core kernels raise if a pipeline wait times out (never expected)."""
    key = (device.type, device.index)
    if key not in _TC_ERR:
        _TC_ERR[key] = torch.zeros(1, dtype=torch.int32, device=device)
    return _TC_ERR[key]


def tc_supported(cin, cout):
    """Channel pairs of the tensor-core scatter-dgrad kernel (`tc_scatter_ch_ok`, csrc/common.cuh)."""
    return cin in (16, 32, 64) and cout in (16, 32, 64)


def tc_conv_supported(cin, cout):
    """Channel pairs of the tensor-core conv forward / gather-dgrad / wgrad kernels (csrc/conv_tc2.cu, csrc/wgrad_tc3.cu):
    the C = 8 layers run with K and N padded to 16 (zero-filled by the gather / the weight image)."""
    return cin in (8, 16, 32, 64) and cout in (8, 16, 32, 64)


def cast_bf16(t):
    """fp32 [N, C] -> bf16 copy (the gathered operand of the tensor-core kernels)."""
    _require_cuda(t)
    lib = _lib.load()
    t = t.contiguous()
    out = torch.empty(t.shape, dtype=torch.bfloat16, device=t.device)
    _timed('cast_bf16', t.numel() * 6, 0,
           lambda: check(lib.vc_cast_f32_bf16(_p(t), _p(out), t.numel(), _stream()), 'vc_cast_f32_bf16'))
    return out


# ------------------------------------------------------------------------------------------------
# rulebooks
# ------------------------------------------------------------------------------------------------
@dataclass
class Rulebook:
    """Neighbour-table rulebook (canonical form: oracle/rulebook.py, SURVEY §8a-R)."""
    subm: bool
    ndim: int
    K: int
    n_in: int
    n_out: int
    nbr: torch.Tensor                      # [K, n_out] int32: input row per (offset, output row) or -1
    nbr_bwd: torch.Tensor | None           # [K, n_in]  int32: output row per (offset, input row) (regular conv)
    pair_num: torch.Tensor                 # [K] int32
    out_indices: torch.Tensor              # [n_out, 1+ndim] int32
    out_shape: list
    unique_coords: bool = True             # False: many-to-one table (image branch) -> scatter dgrad
    _pairs: tuple | None = field(default=None, repr=False)

    def n_pairs(self):
        """total rulebook entries P (host read; only the bench's roofline accounting calls this)."""
        if getattr(self, '_np', None) is None:
            self._np = int(self.pair_num.sum().item())
        return self._np

    def indice_pairs(self):
        """spconv-style (indice_pairs [2,K,n_out], indice_pair_num [K]); built on demand."""
        if self._pairs is None:
            lib = _lib.load()
            pairs = torch.empty((2, self.K, max(self.n_out, 1)), dtype=torch.int32, device=self.nbr.device)
            num = torch.empty((self.K,), dtype=torch.int32, device=self.nbr.device)
            check(lib.vc_pairs_from_nbr(_p(self.nbr), self.K, self.n_out, _p(pairs), _p(num), _stream()),
                  'vc_pairs_from_nbr')
            self._pairs = (pairs[:, :, :self.n_out], num)
        return self._pairs


def build_subm_rulebook(indices, batch_size, spatial_shape, ksize, dilation=1, unique_coords=None) -> Rulebook:
    _require_cuda(indices)
    lib = _lib.load()
    assert indices.dtype == torch.int32 and indices.is_contiguous()
    n, nd = indices.shape[0], indices.shape[1] - 1
    ks, dil = _tup(ksize, nd), _tup(dilation, nd)
    K = int(np.prod(ks))
    nbr = torch.empty((K, n), dtype=torch.int32, device=indices.device)
    pair_num = torch.empty((K,), dtype=torch.int32, device=indices.device)
    ws = _ws(lib.vc_subm_rulebook_ws_bytes(n), indices.device)
    check(lib.vc_subm_rulebook(_p(indices), n, nd, int(batch_size), host_i32(spatial_shape), host_i32(ks),
                               host_i32(dil), _p(nbr), _p(pair_num), _p(ws), ws.numel(), _stream()),
          'vc_subm_rulebook')
    if unique_coords is None:
        unique_coords = nd == 3      # voxel grids are duplicate free; projected image indices are not
    return Rulebook(True, nd, K, n, n, nbr, None, pair_num, indices, list(spatial_shape), unique_coords)


def build_conv_rulebook(indices, batch_size, spatial_shape, ksize, stride, padding, dilation=1) -> Rulebook:
    _require_cuda(indices)
    lib = _lib.load()
    assert indices.dtype == torch.int32 and indices.is_contiguous()
    n, nd = indices.shape[0], indices.shape[1] - 1
    ks, st, pd, dil = _tup(ksize, nd), _tup(stride, nd), _tup(padding, nd), _tup(dilation, nd)
    K = int(np.prod(ks))
    geo = (host_i32(spatial_shape), host_i32(ks), host_i32(st), host_i32(pd), host_i32(dil))
    oshape = host_i32([0] * nd)
    check(lib.vc_conv_out_shape(nd, *geo, oshape), 'vc_conv_out_shape')
    out_shape = [int(v) for v in oshape]
    ws = _ws(lib.vc_conv_rulebook_ws_bytes(nd, int(batch_size), oshape), indices.device)
    n_out_dev = torch.empty((1,), dtype=torch.int32, device=indices.device)
    check(lib.vc_conv_rulebook_count(_p(indices), n, nd, int(batch_size), *geo, _p(n_out_dev), _p(ws), ws.numel(),
                                     _stream()), 'vc_conv_rulebook_count')
    n_out = int(n_out_dev.item())        # the one host read per strided conv (output row count is data dependent)
    out_indices = torch.empty((n_out, 1 + nd), dtype=torch.int32, device=indices.device)
    nbr = torch.empty((K, n_out), dtype=torch.int32, device=indices.device)
    nbr_bwd = torch.empty((K, n), dtype=torch.int32, device=indices.device)
    pair_num = torch.empty((K,), dtype=torch.int32, device=indices.device)
    check(lib.vc_conv_rulebook_fill(_p(indices), n, nd, int(batch_size), *geo, n_out, _p(out_indices), _p(nbr),
                                    _p(nbr_bwd), _p(pair_num), _p(ws), ws.numel(), _stream()),
          'vc_conv_rulebook_fill')
    return Rulebook(False, nd, K, n, n_out, nbr, nbr_bwd, pair_num, out_indices, out_shape, True)


# ------------------------------------------------------------------------------------------------
# raw kernels
# ------------------------------------------------------------------------------------------------
def conv_forward(feats, weight, rb: Rulebook, bn_sums=None, precision='fp32', feats_bf16=None, keep=None):
    """feats [n_in, C_in] f32, weight [C_out, *k, C_in] f32 -> out [n_out, C_out]; when `bn_sums` ([2*C_out] float64,
    zeroed) is given the kernel adds the output's channel sums (sum x, sum x^2) to it."""
    _require_cuda(feats, weight)
    lib = _lib.load()
    cout, cin = weight.shape[0], weight.shape[-1]
    feats = feats.contiguous()
    weight = weight.contiguous()
    out = torch.empty((rb.n_out, cout), dtype=torch.float32, device=feats.device)
    if precision == 'bf16' and tc_conv_supported(cin, cout) and rb.n_out > 0:
        fb = feats_bf16 if feats_bf16 is not None else cast_bf16(feats)
        if keep is not None:
            keep['feats_bf16'] = fb
        ws = _ws(lib.vc_conv_tc_ws_bytes(cin, cout, rb.K), feats.device)
        n_in = feats.shape[0]
        _timed('conv_fwd_tc',
               lambda: n_in * cin * 2 + rb.n_out * cout * 4 + rb.K * cin * cout * 2 + rb.n_pairs() * 8,
               lambda: 2 * rb.n_pairs() * cin * cout,
               lambda: check(lib.vc_conv_fwd_tc(_p(fb), _p(weight), _p(rb.nbr), _p(out), rb.n_out, cin, cout, rb.K,
                                                _p(bn_sums), _p(ws), ws.numel(), _p(tc_error_flag(feats.device)),
                                                _stream()), 'vc_conv_fwd_tc'))
        return out
    ws = _ws(lib.vc_conv_ws_bytes(cin, cout, rb.K), feats.device)
    n_in = feats.shape[0]
    _timed('conv_fwd',
           lambda: (n_in * cin + rb.n_out * cout + rb.K * cin * cout) * 4 + rb.n_pairs() * 8,
           lambda: 2 * rb.n_pairs() * cin * cout,
           lambda: check(lib.vc_conv_fwd_f32(_p(feats), _p(weight), _p(rb.nbr), _p(out), rb.n_out, cin, cout, rb.K,
                                             _p(bn_sums), _p(ws), ws.numel(), _stream()), 'vc_conv_fwd_f32'))
    return out


def conv_dgrad(dout, weight, rb: Rulebook, precision='fp32', dout_bf16=None):
    _require_cuda(dout, weight)
    lib = _lib.load()
    cout, cin = weight.shape[0], weight.shape[-1]
    dout = dout.contiguous()
    weight = weight.contiguous()
    if precision == 'bf16' and tc_conv_supported(cin, cout) and rb.n_in > 0 and not (rb.subm and not rb.unique_coords):
        db = dout_bf16 if dout_bf16 is not None else cast_bf16(dout)
        din = torch.empty((rb.n_in, cin), dtype=torch.float32, device=dout.device)
        table, mirror = (rb.nbr, 1) if rb.subm else (rb.nbr_bwd, 0)
        ws = _ws(lib.vc_conv_tc_ws_bytes(cin, cout, rb.K), dout.device)
        _timed('conv_dgrad_tc',
               lambda: rb.n_out * cout * 2 + rb.n_in * cin * 4 + rb.K * cin * cout * 2 + rb.n_pairs() * 8,
               lambda: 2 * rb.n_pairs() * cin * cout,
               lambda: check(lib.vc_conv_dgrad_tc(_p(db), _p(weight), _p(table), _p(din), rb.n_in, cin, cout, rb.K, mirror,
                                                  _p(ws), ws.numel(), _p(tc_error_flag(dout.device)), _stream()),
                             'vc_conv_dgrad_tc'))
        return din
    if rb.subm and not rb.unique_coords and precision == 'bf16' and tc_supported(cin, cout) and rb.n_out > 0:
        # image branch (many-to-one table): GEMM on the tensor cores, result scattered with vector reductions
        db = dout_bf16 if dout_bf16 is not None else cast_bf16(dout)
        din = torch.zeros((rb.n_in, cin), dtype=torch.float32, device=dout.device)
        ws = _ws(lib.vc_conv_tc_ws_bytes(cin, cout, rb.K), dout.device)
        _timed('conv_dgrad_scatter_tc',
               lambda: rb.n_out * cout * 2 + rb.n_in * cin * 4 + rb.K * cin * cout * 2 + rb.n_pairs() * 8,
               lambda: 2 * rb.n_pairs() * cin * cout,
               lambda: check(lib.vc_conv_dgrad_scatter_tc(_p(db), _p(weight), _p(rb.nbr), _p(din), rb.n_out, cin, cout, rb.K,
                                                          _p(ws), ws.numel(), _p(tc_error_flag(dout.device)), _stream()),
                             'vc_conv_dgrad_scatter_tc'))
        return din
    ws = _ws(lib.vc_conv_ws_bytes(cin, cout, rb.K), dout.device)
    if rb.subm and not rb.unique_coords:
        din = torch.zeros((rb.n_in, cin), dtype=torch.float32, device=dout.device)
        _timed('conv_dgrad_scatter',
               lambda: (rb.n_in * cin + rb.n_out * cout + rb.K * cin * cout) * 4 + rb.n_pairs() * 8,
               lambda: 2 * rb.n_pairs() * cin * cout,
               lambda: check(lib.vc_conv_dgrad_scatter_f32(_p(dout), _p(weight), _p(rb.nbr), _p(din), rb.n_out, cin,
                                                           cout, rb.K, _p(ws), ws.numel(), _stream()),
                             'vc_conv_dgrad_scatter_f32'))
        return din
    din = torch.empty((rb.n_in, cin), dtype=torch.float32, device=dout.device)
    table, mirror = (rb.nbr, 1) if rb.subm else (rb.nbr_bwd, 0)
    _timed('conv_dgrad',
           lambda: (rb.n_in * cin + rb.n_out * cout + rb.K * cin * cout) * 4 + rb.n_pairs() * 8,
           lambda: 2 * rb.n_pairs() * cin * cout,
           lambda: check(lib.vc_conv_dgrad_f32(_p(dout), _p(weight), _p(table), _p(din), rb.n_in, cin, cout, rb.K, mirror,
                                               _p(ws), ws.numel(), _stream()), 'vc_conv_dgrad_f32'))
    return din


def conv_wgrad(feats, dout, weight_shape, rb: Rulebook, precision='fp32', feats_bf16=None, dout_bf16=None):
    _require_cuda(feats, dout)
    lib = _lib.load()
    cout, cin = weight_shape[0], weight_shape[-1]
    feats = feats.contiguous()
    dout = dout.contiguous()
    dw = torch.empty(tuple(weight_shape), dtype=torch.float32, device=feats.device)
    if precision == 'bf16' and tc_conv_supported(cin, cout) and rb.n_out > 0:
        fb = feats_bf16 if feats_bf16 is not None else cast_bf16(feats)
        db = dout_bf16 if dout_bf16 is not None else cast_bf16(dout)
        ws = _ws(lib.vc_conv_wgrad_tc_ws_bytes(rb.n_out, cin, cout, rb.K), feats.device)
        n_in = feats.shape[0]
        _timed('conv_wgrad_tc',
               lambda: (n_in * cin + rb.n_out * cout) * 2 + rb.K * cin * cout * 4 + rb.n_pairs() * 8,
               lambda: 2 * rb.n_pairs() * cin * cout,
               lambda: check(lib.vc_conv_wgrad_tc(_p(fb), _p(db), _p(rb.nbr), _p(dw), rb.n_out, cin, cout, rb.K, _p(ws),
                                                  ws.numel(), _p(tc_error_flag(feats.device)), _stream()),
                             'vc_conv_wgrad_tc'))
        return dw
    ws = _ws(lib.vc_conv_wgrad_ws_bytes(rb.n_out, cin, cout, rb.K), feats.device)
    n_in = feats.shape[0]
    _timed('conv_wgrad',
           lambda: (n_in * cin + rb.n_out * cout + rb.K * cin * cout) * 4 + rb.n_pairs() * 8,
           lambda: 2 * rb.n_pairs() * cin * cout,
           lambda: check(lib.vc_conv_wgrad_f32(_p(feats), _p(dout), _p(rb.nbr), _p(dw), rb.n_out, cin, cout, rb.K, _p(ws),
                                               ws.numel(), _stream()), 'vc_conv_wgrad_f32'))
    return dw


class SparseConvFn(torch.autograd.Function):
    """Plain sparse convolution (no norm): out = conv(feats, weight) through a rulebook."""

    @staticmethod
    def forward(ctx, feats, weight, rb, precision='fp32'):
        keep = {}
        out = conv_forward(feats, weight, rb, None, precision, keep=keep)
        ctx.rb, ctx.precision = rb, precision
        ctx.fb = keep.get('feats_bf16')
        ctx.save_for_backward(feats, weight)
        return out

    @staticmethod
    def backward(ctx, dout):
        feats, weight = ctx.saved_tensors
        rb = ctx.rb
        dout = dout.contiguous()
        cout, cin = weight.shape[0], weight.shape[-1]
        db = cast_bf16(dout) if (ctx.precision == 'bf16' and tc_conv_supported(cin, cout) and rb.n_out > 0) else None
        din = conv_dgrad(dout, weight, rb, ctx.precision, db) if ctx.needs_input_grad[0] else None
        dw = conv_wgrad(feats, dout, weight.shape, rb, ctx.precision, ctx.fb, db) if ctx.needs_input_grad[1] else None
        return din, dw, None, None


class ConvBNReLUFn(torch.autograd.Function):
    """conv -> BatchNorm1d (batch or running statistics) -> ReLU, the unit every VirConv layer is built from
    (spconv_backbone.py:86-131).  BN statistics ride on the conv epilogue; backward = BN/ReLU backward ->
    dgrad + wgrad.  In 'bf16' precision the op also returns a bf16 shadow of its output (non-differentiable) that
    the next layer gathers from, and accepts the shadow of its own input (`feats_bf16`)."""

    @staticmethod
    def forward(ctx, feats, weight, gamma, beta, running_mean, running_var, rb, training, eps, momentum,
                precision='fp32', feats_bf16=None, num_batches_tracked=None):
        lib = _lib.load()
        ctx.set_materialize_grads(False)
        dev = feats.device
        cout = weight.shape[0]
        keep = {}
        sums = stats_arena(dev).take(4 * cout)      # [0:2C] forward sums, [2C:4C] backward sums (used in backward)
        x = conv_forward(feats, weight, rb, sums if training else None, precision, feats_bf16=feats_bf16, keep=keep)
        ctx.fb = keep.get('feats_bf16')
        stats = torch.empty((4, cout), dtype=torch.float32, device=dev)  # scale, shift, mean, invstd
        y = torch.empty_like(x)
        yb = torch.empty(x.shape, dtype=torch.bfloat16, device=dev) if precision == 'bf16' else None
        check(lib.vc_bn_apply_relu_f32(_p(x), _p(sums), rb.n_out, cout, _p(gamma), _p(beta), _p(running_mean),
                                       _p(running_var), _p(num_batches_tracked), float(momentum), float(eps), int(training),
                                       _p(y), _p(yb), _p(stats), 1, _stream()), 'vc_bn_apply_relu_f32')
        ctx.bsums, ctx.arena_gen = sums[2 * cout:], stats_arena(dev).generation
        ctx.rb, ctx.training, ctx.precision = rb, training, precision
        ctx.save_for_backward(feats, weight, gamma, x, y, stats)
        if yb is None:
            return y
        ctx.mark_non_differentiable(yb)
        return y, yb

    @staticmethod
    def backward(ctx, dy, *unused):
        lib = _lib.load()
        feats, weight, gamma, x, y, stats = ctx.saved_tensors
        rb = ctx.rb
        cout, cin = weight.shape[0], weight.shape[-1]
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        use_tc = ctx.precision == 'bf16' and tc_conv_supported(cin, cout) and rb.n_out > 0
        db = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device) if use_tc else None
        dgamma = torch.empty_like(gamma)
        dbeta = torch.empty_like(gamma)
        bsums = ctx.bsums
        if stats_arena(dy.device).generation != ctx.arena_gen:     # another forward re-used the arena since: own zeros
            bsums = torch.zeros(2 * cout, dtype=torch.float64, device=dy.device)
        check(lib.vc_bn_relu_bwd_f32(_p(dy), _p(x), _p(y), _p(gamma), _p(stats), _p(dx), _p(db), _p(dgamma), _p(dbeta),
                                     rb.n_out, cout, int(ctx.training), _p(bsums), _stream()), 'vc_bn_relu_bwd_f32')
        dw = conv_wgrad(feats, dx, weight.shape, rb, ctx.precision, ctx.fb, db) if ctx.needs_input_grad[1] else None
        din = conv_dgrad(dx, weight, rb, ctx.precision, db) if ctx.needs_input_grad[0] else None
        return din, dw, dgamma, dbeta, None, None, None, None, None, None, None, None, None


class Cat2Fn(torch.autograd.Function):
    """Channel concat of the 3-D and 2-D branch outputs of an NRConv block (spconv_backbone.py:227), optionally with
    the bf16 shadow of the result (the next strided conv's tensor-core operand)."""

    @staticmethod
    def forward(ctx, a, b, want_bf16):
        _require_cuda(a, b)
        lib = _lib.load()
        ctx.set_materialize_grads(False)
        a, b = a.contiguous(), b.contiguous()
        n, ca, cb = a.shape[0], a.shape[1], b.shape[1]
        out = torch.empty((n, ca + cb), dtype=torch.float32, device=a.device)
        ob = torch.empty((n, ca + cb), dtype=torch.bfloat16, device=a.device) if want_bf16 else None
        check(lib.vc_cat2_f32(_p(a), _p(b), _p(out), _p(ob), n, ca, cb, _stream()), 'vc_cat2_f32')
        ctx.ca = ca
        if ob is None:
            return out
        ctx.mark_non_differentiable(ob)
        return out, ob

    @staticmethod
    def backward(ctx, dout, *unused):
        return dout[:, :ctx.ca], dout[:, ctx.ca:], None


# ------------------------------------------------------------------------------------------------
# voxel index -> pixel index
# ------------------------------------------------------------------------------------------------
def _f32(x):
    return np.float32(x)


def compose_lidar_to_rect(V2C, R0):
    """M[4,3] = V2C^T @ R0^T in float32, left-to-right multiply/add (the order the kernel and the oracle share;
    the reference lets torch.matmul pick it, calibration_kitti.py:126-128)."""
    a = np.asarray(V2C, dtype=np.float32).T
    b = np.asarray(R0, dtype=np.float32).T
    m = np.zeros((4, 3), dtype=np.float32)
    for i in range(4):
        for j in range(3):
            m[i, j] = _f32(_f32(_f32(a[i, 0] * b[0, j]) + _f32(a[i, 1] * b[1, j])) + _f32(a[i, 2] * b[2, j]))
    return m


def projection_params_host(calib, trans_param, batch_size):
    """[B, 28] float32 parameter block of vc_index2uv (layout: include/virconv_b200.h) as a numpy array."""
    tp = None
    if trans_param is not None:
        tp = trans_param.detach().cpu().numpy() if torch.is_tensor(trans_param) else np.asarray(trans_param)
        tp = tp.astype(np.float32)
    out = np.zeros((batch_size, 28), dtype=np.float32)
    for b in range(batch_size):
        cached = getattr(calib[b], '_vc_proj20', None)      # a Calibration object is immutable after construction
        if cached is None:
            cached = np.concatenate([compose_lidar_to_rect(calib[b].V2C, calib[b].R0).reshape(-1),
                                     np.asarray(calib[b].P2, dtype=np.float32).T[:, :2].reshape(-1)])
            try:
                calib[b]._vc_proj20 = cached
            except AttributeError:
                pass
        out[b, 0:20] = cached
        if tp is not None:
            rot, flip, scale = tp[b]
            out[b, 20] = 1.0
            out[b, 21] = scale
            out[b, 22] = flip
            out[b, 23] = np.cos(_f32(-rot))
            out[b, 24] = np.sin(_f32(-rot))
    return out


def projection_params(calib, trans_param, batch_size, device, stream=None):
    """The block of projection_params_host on the device.  `stream`: upload on that torch stream (the plan executor
    consumes the block on its side stream only)."""
    out = projection_params_host(calib, trans_param, batch_size)
    if stream is not None:
        with torch.cuda.stream(stream):
            return torch.from_numpy(out).to(device, non_blocking=True)
    return torch.from_numpy(out).to(device, non_blocking=True)


def index2uv(indices, batch_size, params, stride, pts_range=(0, -40, -3, 70.4, 40, 1),
             voxel_size=(0.05, 0.05, 0.05), u_max=1400, v_max=600):
    """(b, z, y, x) int32 -> (b, u//stride, v//stride) int32; arithmetic of spconv_backbone.py:8-24,54-83."""
    _require_cuda(indices, params)
    lib = _lib.load()
    assert indices.dtype == torch.int32 and indices.shape[1] == 4 and indices.is_contiguous()
    vs = np.array(voxel_size, dtype=np.float64) * stride
    grid = host_f32([vs[0], vs[1], vs[2], pts_range[0] + vs[0] / 2, pts_range[1] + vs[1] / 2,
                     pts_range[2] + vs[2] / 2])
    uv = torch.empty((indices.shape[0], 3), dtype=torch.int32, device=indices.device)
    check(lib.vc_index2uv(_p(indices), indices.shape[0], int(batch_size), _p(params), grid, int(stride), u_max, v_max,
                          _p(uv), _stream()), 'vc_index2uv')
    return uv


# ------------------------------------------------------------------------------------------------
# dense / gather
# ------------------------------------------------------------------------------------------------
class DenseFn(torch.autograd.Function):
    """`SparseConvTensor.dense()`.  num_rows (device int32[1], may be None): the valid rows of a static-mode tensor whose
    features / indices are capacity sized (vc_dense_rows_f32: the -1 index tail is never scattered, its gradient is zero)."""

    @staticmethod
    def forward(ctx, feats, indices, batch_size, spatial_shape, num_rows=None):
        _require_cuda(feats, indices, num_rows)
        lib = _lib.load()
        n, c = feats.shape
        nd = indices.shape[1] - 1
        out = torch.zeros((batch_size, c, *spatial_shape), dtype=torch.float32, device=feats.device)
        if num_rows is None:
            check(lib.vc_dense_f32(_p(feats.contiguous()), _p(indices), n, c, nd, int(batch_size), host_i32(spatial_shape),
                                   _p(out), _stream()), 'vc_dense_f32')
        else:
            assert num_rows.dtype == torch.int32 and num_rows.numel() == 1 and indices.shape[0] == n
            check(lib.vc_dense_rows_f32(_p(feats.contiguous()), _p(indices), n, _p(num_rows), c, nd, int(batch_size),
                                        host_i32(spatial_shape), _p(out), _stream()), 'vc_dense_rows_f32')
        ctx.save_for_backward(indices)
        ctx.num_rows = num_rows
        ctx.meta = (n, c, nd, int(batch_size), list(spatial_shape))
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = _lib.load()
        (indices,) = ctx.saved_tensors
        n, c, nd, bs, shape = ctx.meta
        df = torch.empty((n, c), dtype=torch.float32, device=dout.device)
        if ctx.num_rows is None:
            check(lib.vc_dense_bwd_f32(_p(dout.contiguous()), _p(indices), n, c, nd, bs, host_i32(shape), _p(df), _stream()),
                  'vc_dense_bwd_f32')
        else:
            check(lib.vc_dense_rows_bwd_f32(_p(dout.contiguous()), _p(indices), n, _p(ctx.num_rows), c, nd, bs, host_i32(shape),
                                            _p(df), _stream()), 'vc_dense_rows_bwd_f32')
        return df, None, None, None, None


def gather_rows(t, rows):
    """out[r] = t[rows[r]] (StVD layer discard, spconv_backbone.py:134-147); rows int32 on device."""
    _require_cuda(t, rows)
    lib = _lib.load()
    t = t.contiguous()
    out = torch.empty((rows.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    row_bytes = t.element_size() * int(np.prod(t.shape[1:]))
    check(lib.vc_gather_rows(_p(t), _p(rows), _p(out), rows.shape[0], row_bytes, _stream()), 'vc_gather_rows')
    return out


class GatherRowsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feats, rows):
        ctx.save_for_backward(rows)
        ctx.n = feats.shape[0]
        return gather_rows(feats, rows)

    @staticmethod
    def backward(ctx, dout):
        (rows,) = ctx.saved_tensors
        din = torch.zeros((ctx.n, dout.shape[1]), dtype=dout.dtype, device=dout.device)
        din.index_copy_(0, rows.long(), dout.contiguous())   # rows are unique (a subsample)
        return din, None


def stvd_layer_keep(n, rate, site, seed=None, keys=None, n_dev=None, device=None):
    """Device-drawn StVD layer discard rows (vc_stvd_layer_keep): over n rows (n_dev: device int32[1] of valid rows, n
    the capacity), the k = int(n_valid * (1 - rate)) rows with the smallest (Philox key of (row, site) under `seed`, row),
    or of the given uint32 `keys` (an int64 / int32 tensor holding them), ascending.  -> (keep [n] int32 with a -1 tail,
    kept [1] int32, pos [n] int32 = position in keep or -1)."""
    lib = _lib.load()
    dev = torch.device(device) if device is not None else (seed if seed is not None else keys).device
    n = int(n)
    keep = torch.empty((n,), dtype=torch.int32, device=dev)
    pos = torch.empty((n,), dtype=torch.int32, device=dev)
    kept = torch.empty((1,), dtype=torch.int32, device=dev)
    if keys is not None:
        keys = keys.to(device=dev, dtype=torch.int64).to(torch.int32).contiguous()     # (bit pattern of the uint32 keys)
        assert keys.numel() >= n
    if seed is not None:
        assert seed.dtype == torch.int64 and seed.device == dev
    ws = _ws(lib.vc_stvd_layer_keep_ws_bytes(n), dev)
    check(lib.vc_stvd_layer_keep(_p(keys), _p(seed), int(site), n, _p(n_dev), float(rate), _p(keep), _p(kept), _p(pos), _p(ws),
                                 ws.numel(), _stream()), 'vc_stvd_layer_keep')
    return keep, kept, pos


# ------------------------------------------------------------------------------------------------
# voxelisation + MeanVFE, voxel -> row map
# ------------------------------------------------------------------------------------------------
def voxelize_mean(points, batch_size, pc_range=(0, -40, -3, 70.4, 40, 1), voxel_size=(0.05, 0.05, 0.05), max_points=5,
                  max_voxels=40000, vfe_model='max', want_voxels=False, static=False):
    """points [N, 1+C] f32 (b, x, y, z, ...), batch-contiguous -> (voxel_features [M,C], voxel_coords [M,4] int32
    (b,z,y,x), voxel_num_points [M] int32[, voxels [M,max_points,C]]): the dataloader's first-come voxeliser
    (data_processor.py:43-59) fused with MeanVFE (mean_vfe.py:39-58), on the GPU.
    static=True (CUDA-graph capturable): no host read of the voxel count — returns capacity-sized tensors
    (batch_size * max_voxels rows, zero / -1 tail) plus the count as a device int32[1] tensor; `points` may then be a
    capacity-sized buffer whose unused tail rows carry out-of-range coordinates (they are dropped like any such point)."""
    _require_cuda(points)
    lib = _lib.load()
    points = points.contiguous()
    n, c = points.shape[0], points.shape[1] - 1
    cap = int(batch_size) * int(max_voxels)
    dev = points.device
    if static:
        feats = torch.zeros((cap, c), dtype=torch.float32, device=dev)
        coords = torch.full((cap, 4), -1, dtype=torch.int32, device=dev)
        num = torch.zeros((cap,), dtype=torch.int32, device=dev)
    else:
        feats = torch.empty((cap, c), dtype=torch.float32, device=dev)
        coords = torch.empty((cap, 4), dtype=torch.int32, device=dev)
        num = torch.empty((cap,), dtype=torch.int32, device=dev)
    voxels = torch.zeros((cap, max_points, c), dtype=torch.float32, device=dev) if want_voxels else None
    n_out = torch.empty((1,), dtype=torch.int32, device=dev)
    ws = _ws(lib.vc_voxelize_ws_bytes(n, int(batch_size), int(max_points)), dev)
    check(lib.vc_voxelize_mean(_p(points), n, c, int(batch_size), host_f32(pc_range), host_f32(voxel_size), int(max_points),
                               int(max_voxels), int(vfe_model == 'max'), _p(feats), _p(coords), _p(num), _p(voxels),
                               _p(n_out), _p(ws), ws.numel(), _stream()), 'vc_voxelize_mean')
    if static:
        return (feats, coords, num, n_out) + ((voxels,) if want_voxels else ())
    m = int(n_out.item())
    out = (feats[:m], coords[:m], num[:m])
    return out + (voxels[:m],) if want_voxels else out


def voxel2pinds(indices, batch_size, spatial_shape, num_rows=None):
    """Dense voxel -> row map (`generate_voxel2pinds`, pcdet/utils/spconv_utils.py:13-21).  num_rows (device int32[1]): the
    valid rows of a static-mode tensor's capacity-sized indices (`t.num_rows`); the -1 tail is skipped."""
    _require_cuda(indices, num_rows)
    lib = _lib.load()
    indices = indices.to(torch.int32).contiguous()
    out = torch.empty((int(batch_size), *[int(s) for s in spatial_shape]), dtype=torch.int32, device=indices.device)
    if num_rows is None:
        check(lib.vc_voxel2pinds(_p(indices), indices.shape[0], indices.shape[1] - 1, int(batch_size), host_i32(spatial_shape),
                                 _p(out), _stream()), 'vc_voxel2pinds')
        return out
    assert num_rows.dtype == torch.int32 and num_rows.numel() == 1
    check(lib.vc_voxel2pinds_rows(_p(indices), indices.shape[0], _p(num_rows), indices.shape[1] - 1, int(batch_size),
                                  host_i32(spatial_shape), _p(out), _stream()), 'vc_voxel2pinds_rows')
    return out


# ------------------------------------------------------------------------------------------------
# test-time x-batching of the ROT_NUM transformed copies (csrc/xbatch.cu)
# ------------------------------------------------------------------------------------------------
XBATCH_MAX = 4          # the reference batches at most 4 copies along x (spconv_backbone.py:360)


def xbatch_pack(feats, coords, counts, width, n_out=None):
    """R <= 4 capacity-sized copies (features [cap_i, C] fp32, coordinates [cap_i, 4] int32, device int32[1] row counts) ->
    (features [sum cap_i, C], coordinates [sum cap_i, 4], n_out): the valid rows of copy 0, copy 1, ... in order with
    x += i * width (torch.cat of the exact rows), zero / -1 tail; n_out (given or fresh) receives the total row count."""
    R = len(feats)
    if not 1 <= R <= XBATCH_MAX or len(coords) != R or len(counts) != R:
        raise ValueError('xbatch_pack: 1..%d copies, one coordinate tensor and count each (got %d, %d, %d)'
                         % (XBATCH_MAX, R, len(coords), len(counts)))
    _require_cuda(*feats, *coords, *counts)
    lib = _lib.load()
    feats = [f.contiguous() for f in feats]
    for f, c, n in zip(feats, coords, counts):
        assert f.dtype == torch.float32 and f.shape[1] == feats[0].shape[1], (f.dtype, f.shape)
        assert c.dtype == torch.int32 and c.is_contiguous() and c.shape == (f.shape[0], 4), (c.dtype, c.shape)
        assert n.dtype == torch.int32 and n.numel() == 1
    dev, C = feats[0].device, feats[0].shape[1]
    cap = sum(f.shape[0] for f in feats)
    out_f = torch.empty((cap, C), dtype=torch.float32, device=dev)
    out_c = torch.empty((cap, 4), dtype=torch.int32, device=dev)
    if n_out is None:
        n_out = torch.empty((1,), dtype=torch.int32, device=dev)
    assert n_out.dtype == torch.int32 and n_out.numel() == 1 and n_out.device == dev
    check(lib.vc_xbatch_pack(_lib.host_ptrs([f.data_ptr() for f in feats]), _lib.host_ptrs([c.data_ptr() for c in coords]),
                             _lib.host_ptrs([n.data_ptr() for n in counts]), host_i32([f.shape[0] for f in feats]), R, C,
                             int(width), cap, _p(out_f), _p(out_c), _p(n_out), _stream()), 'vc_xbatch_pack')
    return out_f, out_c, n_out


def xbatch_split(feats, indices, num_rows, width, R):
    """The device form of backbone.decompose_tensor for all R copies at once: a capacity-sized tensor (features [cap, C] fp32,
    indices [cap, 4] int32, device int32[1] row count) over a grid of x extent `width` -> R (features, indices, num_rows),
    each of capacity cap: copy i holds the rows with i*q < x < (i+1)*q, q = width // 4, in order, x -= i*q; zero / -1 tail."""
    if not 1 <= R <= XBATCH_MAX:
        raise ValueError('xbatch_split: 1..%d copies, got %d' % (XBATCH_MAX, R))
    _require_cuda(feats, indices, num_rows)
    lib = _lib.load()
    feats = feats.contiguous()
    assert feats.dtype == torch.float32 and indices.dtype == torch.int32 and indices.is_contiguous()
    assert indices.shape == (feats.shape[0], 4) and num_rows.dtype == torch.int32 and num_rows.numel() == 1
    cap, C, dev = feats.shape[0], feats.shape[1], feats.device
    outs = [(torch.empty((cap, C), dtype=torch.float32, device=dev), torch.empty((cap, 4), dtype=torch.int32, device=dev),
             torch.empty((1,), dtype=torch.int32, device=dev)) for _ in range(R)]
    ws = _ws(lib.vc_xbatch_split_ws_bytes(cap, R), dev)
    check(lib.vc_xbatch_split(_p(feats), _p(indices), cap, _p(num_rows), C, int(width), R,
                              _lib.host_ptrs([o[0].data_ptr() for o in outs]), _lib.host_ptrs([o[1].data_ptr() for o in outs]),
                              _lib.host_ptrs([o[2].data_ptr() for o in outs]), _p(ws), ws.numel(), _stream()),
          'vc_xbatch_split')
    return outs
