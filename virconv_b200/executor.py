"""Plan executor front end: describe a backbone's layer graph once, run its whole forward / backward through ONE
C-ABI call each (`vc_exec_forward` / `vc_exec_backward`, include/virconv_b200.h; host loop in csrc/executor.cu).

The reference walks the backbone layer by layer in Python (`VirConvL8x.forward` spconv_backbone.py:609-699,
`NRConvBlock.forward` :207-229, `VirConv8x.forward` :339-535) and autograd walks it back; that host work can take
longer than the kernels it launches.  `Plan` records the same graph as a flat op list; `run_plan` executes it natively
and returns ordinary tensors (features with autograd history, indices) that live in one arena allocated per step.
"""
from __future__ import annotations

import copy
import ctypes
import os
import weakref

import numpy as np
import torch

from . import _lib, ops, sync_bn
from ._lib import check

ENABLED = os.environ.get('VIRCONV_EXECUTOR', '1') != '0'
TWO_STREAMS = os.environ.get('VIRCONV_EXEC_STREAMS', '3') != '1'
THREE_STREAMS = os.environ.get('VIRCONV_EXEC_STREAMS', '3') == '3'
# weight gradients on their own stream next to the BN-backward / dgrad chain (vc_exec_backward's wgrad_stream)
WGRAD_STREAM = os.environ.get('VIRCONV_WGRAD_STREAM', '1') != '0'
_WSTREAM = {}


def _wgrad_stream(device):
    if not WGRAD_STREAM:
        return None
    key = (device.type, device.index)
    if key not in _WSTREAM:
        _WSTREAM[key] = torch.cuda.Stream(device=device)
    return _WSTREAM[key]


TIMING = False                     # bench.py's roofline pass: per-launch events around the conv kernels
LAST_RUN = None                    # the most recent forward's record while TIMING is on (bench.py reads its row counts)

OP_SUBM_RB, OP_CONV_RB, OP_INDEX2UV, OP_CBR, OP_CAT, OP_DISCARD = 1, 2, 3, 4, 5, 6
VC_ERR_WORKSPACE = -3
OPI, OPF, PCOLS = 24, 8, 9
# the timing records' kinds: enum ConvKind of csrc/executor.cu
KIND_NAMES = {0: 'conv_fwd', 1: 'conv_fwd_tc', 2: 'conv_dgrad', 3: 'conv_dgrad_tc', 4: 'conv_dgrad_scatter',
              5: 'conv_wgrad', 6: 'conv_wgrad_tc', 7: 'conv_dgrad_scatter_tc', 8: 'conv_dgrad_gather2d',
              9: 'conv_dgrad_gather2d_tc'}


def _t3(v, nd, fill):
    v = list(v) if isinstance(v, (list, tuple)) else [v] * nd
    assert len(v) == nd
    return [int(x) for x in v] + [fill] * (3 - nd)


class Plan:
    """Flat op list over numbered feature slots / index sets / rulebooks (slot 0 / set 0 = the network input)."""

    def __init__(self, in_channels):
        self.rows_i, self.rows_f = [], []
        self.layers = []              # (conv module, bn module)
        self.owners = []              # per layer: the SparseSequential the pair came from (or None)
        self.n_f, self.n_i, self.n_rb = 1, 1, 0
        self.f_channels = {0: in_channels}
        self.published = []           # (name, feature slot, index set)
        self.rb_keys = {}             # rulebook id -> (indice_keys, ndim, in index set, out index set)
        self.discards = []            # (site, op index) of the StVD layer discards, in plan order
        # index set -> group: the sets derived from one another without a layer discard in between.  A published tensor's
        # indice_dict holds the rulebooks of its group only (a discard's output starts a new group, as the module path starts
        # a new SparseConvTensor there), never one built over rows the tensor does not carry
        self.iset_group = {0: 0}
        self.no_grad = {0}            # feature slots no parameter gradient flows into (the input and discards of it)
        self._final = None
        self._slots = None
        # per-device run-time state (dies with the plan, i.e. with the model that owns it)
        self.arena_bytes = {}         # (device index, training) -> arena size handed out (monotone)
        self.arena_used = {}          # (device index, training) -> largest number of arena bytes a step really used
        self.reserved = {}            # (device, stream) -> arena size already parked in the allocator pool
        self.inflight = {}            # device index -> tail events of the forwards still in flight

    # a plan is a cache derived from the modules: copies / pickles of the owning model drop it and rebuild it lazily
    def __deepcopy__(self, memo):
        return None

    def __reduce__(self):
        return (type(None), ())

    def _row(self, kind, stream, a=0, b=0, c=0, ndim=0, ks=(0, 0, 0), st=(1, 1, 1), pd=(0, 0, 0), dl=(1, 1, 1), cin=0,
             cout=0, layer=0, x0=0, x1=0, x2=0, f=()):
        self.rows_i.append([kind, stream, a, b, c, ndim, *ks, *st, *pd, *dl, cin, cout, layer, x0, x1, x2])
        self.rows_f.append(list(f) + [0.0] * (OPF - len(f)))
        self._final = None
        self._slots = None

    def subm_rb(self, iset, ndim, ksize, dilation=1, unique=True, keys=(), stream=1):
        """stream: 1 = index stream, 2 = second index stream (the image branch: its projection + 2-D rulebooks depend on a
        stage's indices only, so they run beside the 3-D rulebooks of the same and the following stages)"""
        rb = self.n_rb
        self.n_rb += 1
        self.rb_keys[rb] = (tuple(keys), ndim, iset, iset)
        self._row(OP_SUBM_RB, stream, a=iset, c=rb, ndim=ndim, ks=_t3(ksize, ndim, 1), dl=_t3(dilation, ndim, 1), x0=int(unique))
        return rb

    def conv_rb(self, iset, ndim, ksize, stride, padding, dilation=1, keys=()):
        rb, out = self.n_rb, self.n_i
        self.n_rb += 1
        self.n_i += 1
        self.rb_keys[rb] = (tuple(keys), ndim, iset, out)
        self.iset_group[out] = self.iset_group[iset]
        self._row(OP_CONV_RB, 1, a=iset, b=out, c=rb, ndim=ndim, ks=_t3(ksize, ndim, 1), st=_t3(stride, ndim, 1),
                  pd=_t3(padding, ndim, 0), dl=_t3(dilation, ndim, 1))
        return out, rb

    def index2uv(self, iset, stride, pts_range=(0, -40, -3, 70.4, 40, 1), voxel_size=(0.05, 0.05, 0.05), u_max=1400,
                 v_max=600, image_shape=(1600, 600), stream=1):
        out = self.n_i
        self.n_i += 1
        self.iset_group[out] = self.iset_group[iset]
        vs = np.array(voxel_size, dtype=np.float64) * stride      # same host arithmetic as ops.index2uv
        grid = [vs[0], vs[1], vs[2], pts_range[0] + vs[0] / 2, pts_range[1] + vs[1] / 2, pts_range[2] + vs[2] / 2]
        self._row(OP_INDEX2UV, stream, a=iset, b=out, ndim=3, ks=(int(image_shape[0]), int(image_shape[1]), 0), x0=int(stride),
                  x1=int(u_max), x2=int(v_max), f=[float(np.float32(g)) for g in grid])
        return out

    def cbr(self, f_in, rb, conv, bn, seq=None):
        """`seq`: the container whose members [0], [1] the (conv, bn) pair was read from — lets is_current() notice a
        swapped sub-module (e.g. SyncBatchNorm.convert_sync_batchnorm after the plan was built, tools/train.py:115-116)."""
        out = self.n_f
        self.n_f += 1
        layer = len(self.layers)
        self.layers.append((conv, bn))
        self.owners.append(seq)
        assert self.f_channels[f_in] == conv.in_channels, (self.f_channels[f_in], conv.in_channels)
        self.f_channels[out] = conv.out_channels
        self._row(OP_CBR, 0, a=f_in, b=out, c=rb, cin=conv.in_channels, cout=conv.out_channels, layer=layer,
                  x0=int(f_in not in self.no_grad))
        return out

    def cat(self, fa, fb):
        out = self.n_f
        self.n_f += 1
        self.f_channels[out] = self.f_channels[fa] + self.f_channels[fb]
        self._row(OP_CAT, 0, a=fa, b=fb, c=out)
        return out

    def discard(self, f, iset, site, rate):
        """StVD layer discard (`layer_voxel_discard`, spconv_backbone.py:134-147) of feature slot `f` over index set `iset`
        at discard site `site`: -> (feature slot, index set) of the kept rows.  The rate reaches the executor as float64 (two
        int32 halves of the op row): int(n * (1 - rate)) must round as Python's does."""
        out_f, out_i = self.n_f, self.n_i
        self.n_f += 1
        self.n_i += 1
        self.f_channels[out_f] = self.f_channels[f]
        self.iset_group[out_i] = max(self.iset_group.values()) + 1
        if f in self.no_grad:
            self.no_grad.add(out_f)
        lo, hi = (int(v) for v in np.array([rate], dtype=np.float64).view(np.int32))
        self.discards.append((int(site), len(self.rows_i)))
        self._row(OP_DISCARD, 1, a=iset, b=out_i, c=int(site), ks=(lo, hi, 0), cin=f, cout=out_f)
        return out_f, out_i

    def publish(self, name, f_slot, iset):
        """The op producing `f_slot` is marked (x1 = 1): its fp32 output is read outside the plan.  The executor writes fp32
        activations only where such a reader exists; the bf16 kernels read the bf16 shadow."""
        self.published.append((name, f_slot, iset))
        for row in self.rows_i:
            if ((row[0] == OP_CBR and row[3] == f_slot) or (row[0] == OP_CAT and row[4] == f_slot)
                    or (row[0] == OP_DISCARD and row[19] == f_slot)):
                row[22] = 1
        self._final = None

    def slot_isets(self):
        """{feature slot: the index set whose rows it holds}"""
        out = {0: 0}
        for r in self.rows_i:
            if r[0] == OP_CBR:
                out[r[3]] = self.rb_keys[r[4]][3]
            elif r[0] == OP_CAT:
                out[r[4]] = out[r[2]]
            elif r[0] == OP_DISCARD:
                out[r[19]] = r[3]
        return out

    def finalize(self):
        if self._final is None:
            oi = np.ascontiguousarray(np.array(self.rows_i, dtype=np.int32).reshape(-1, OPI))
            of = np.ascontiguousarray(np.array(self.rows_f, dtype=np.float32).reshape(-1, OPF))
            lf = np.ascontiguousarray(np.array([[bn.eps, 0.0 if bn.momentum is None else bn.momentum] for _, bn in self.layers],
                                               dtype=np.float32).reshape(-1, 2))
            sizes = []
            for conv, bn in self.layers:
                sizes += [conv.weight.numel(), bn.weight.numel(), bn.bias.numel()]
            offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
            self._final = (oi, of, lf, sizes, offs)
        return self._final

    def params(self):
        out = []
        for conv, bn in self.layers:
            out += [conv.weight, bn.weight, bn.bias]
        return out

    def sync_slots(self):
        """SyncBatchNorm exchange layout (vc_exec_forward_sync): -> (int64 [n_layers, 2] offsets in float64 elements of each
        layer's forward slot [sum x (C), sum x^2 (C), rows] and backward slot [sum g (C), sum g*xhat (C)], total elements).
        The slots of a layer are adjacent, layers follow in plan order."""
        if self._slots is None:
            off, rows = 0, []
            for conv, _ in self.layers:
                c = conv.out_channels
                rows.append([off, off + 2 * c + 1])
                off += 4 * c + 1
            self._slots = (np.ascontiguousarray(np.array(rows, dtype=np.int64).reshape(-1, 2)), off)
        return self._slots

    def eligible(self):
        """Every layer is conv(bias=False) + a plain affine BatchNorm1d or SyncBatchNorm with running statistics and a fixed
        momentum (what the VirConv blocks build, or convert_sync_batchnorm makes of them), all parameters / buffers fp32 and
        contiguous, and SyncBatchNorm layers all of them on one process group.  A cumulative-average BatchNorm
        (momentum=None) or a half-precision model goes through the module path instead."""
        def f32(*ts):
            return all(t is not None and t.dtype == torch.float32 and t.is_contiguous() for t in ts)
        try:
            sync_bn.group_of([bn for _, bn in self.layers])
        except ValueError:
            return False
        return all(conv.bias is None and type(bn) in (torch.nn.BatchNorm1d, torch.nn.SyncBatchNorm) and bn.affine
                   and bn.track_running_stats and bn.momentum is not None
                   and f32(conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var)
                   for conv, bn in self.layers)

    def is_current(self):
        """The (conv, bn) objects recorded at build time are still the live members of their containers."""
        for (conv, bn), seq in zip(self.layers, self.owners):
            if seq is not None and (seq[0] is not conv or seq[1] is not bn):
                return False
        return True


_PINNED = {}


def _pinned(device):
    key = (device.type, device.index)
    if key not in _PINNED:
        _PINNED[key] = torch.empty(16, dtype=torch.int32).pin_memory()
    return _PINNED[key]


ARENA_GRAIN = 64 << 20


def _arena_bytes(plan, n0, device, with_bwd=True, headroom=1.3):
    """Arena size for a step.  First use of a plan: a generous guess from the input row count (VirConv-L uses ~16 KB per
    input voxel, forward + backward; a forward alone about half).  Afterwards: the largest bytes-per-input-row an earlier
    step of the same plan really used (recorded by the backward / the eval forward) times this step's rows plus 30 %
    head-room — monotone per plan, so the caching allocator keeps handing back the same block, and an eval-only or
    small-batch user does not reserve the training worst case (ADVICE r1: rows*24 KB + 256 MB over-reserved ~2x).  `headroom`:
    the factor over the largest use seen (larger under a SyncBatchNorm exchange, which cannot re-run a walk that ran out)."""
    key = (device.index, bool(with_bwd))
    per_row = plan.arena_used.get(key, 0.0)
    if per_row:
        want = int(headroom * per_row * int(n0)) + (32 << 20)
    else:
        # (fixed part: bitmaps / hash tables / weight images / per-layer scratch do not shrink with the batch — a 14 k-voxel
        #  training step uses 540 MB, an 80 k-voxel one 1.1 GB)
        want = int(n0) * (24576 if with_bwd else 12288) + ((384 if with_bwd else 192) << 20)
    want = max(want, plan.arena_bytes.get(key, 0))
    want = (want + ARENA_GRAIN - 1) // ARENA_GRAIN * ARENA_GRAIN
    plan.arena_bytes[key] = want
    return want


def _note_arena_use(plan, device, with_bwd, used, n0):
    key = (device.index, bool(with_bwd))
    plan.arena_used[key] = max(plan.arena_used.get(key, 0.0), float(used) / max(int(n0), 1))


MAX_STEPS_AHEAD = 4          # the host never enqueues more than this many forwards of a plan beyond the GPU
ARENAS_IN_FLIGHT = MAX_STEPS_AHEAD + 3   # (+1 for the step being enqueued, +2: a block handed to three streams with record_stream
                                         #  returns to the pool only after all of them passed it — a cudaMalloc of a multi-GB arena
                                         #  inside a timed loop costs tens of milliseconds)


def _throttle(plan, dev):
    """Bound how far the host runs ahead of the GPU.  Without a per-step synchronisation the only brake is the driver's
    launch-queue depth, and with the step's work spread over four streams that allowed more steps in flight than
    ARENAS_IN_FLIGHT — the next arena then cost a multi-GB cudaMalloc (a 30-100 ms stall once every few runs).  Each
    forward leaves an event at its tail; before a new forward starts, the host waits for the one MAX_STEPS_AHEAD steps
    back (free when the GPU is the bottleneck: the host would otherwise sit in a full launch queue anyway)."""
    q = plan.inflight.setdefault(dev.index, [])
    while len(q) >= MAX_STEPS_AHEAD:
        q.pop(0).synchronize()
    return q


def empty_scratch(n, dtype, dev):
    """torch.empty for library-owned scratch (arenas, the flat gradient buffer) whose every read element the library writes
    first.  Under torch.use_deterministic_algorithms torch would fill the block with NaN on the CURRENT stream; an arena
    belongs to a side stream while the main stream writes it too, so that fill would race with the main stream's first
    writes (and cost a pass over gigabytes per step)."""
    import torch.utils.deterministic as tud
    fill = tud.fill_uninitialized_memory
    tud.fill_uninitialized_memory = False
    try:
        return torch.empty(n, dtype=dtype, device=dev)
    finally:
        tud.fill_uninitialized_memory = fill


def _alloc_arena(plan, nbytes, dev, stream):
    """One arena for this step.  The host may run several steps ahead of the GPU (no per-step synchronisation), so that
    many arenas are alive at once; a fresh multi-GB block costs a cudaMalloc of tens of milliseconds when it lands in
    the middle of training (seen as 5-10 ms/step outliers).  The first time a (plan, size) is used, ARENAS_IN_FLIGHT
    blocks are therefore allocated and released at once, which parks them in the caching allocator's pool of `stream`;
    every later request is served from there."""
    key = (dev.index, stream.cuda_stream if stream is not None else 0)
    ctx = torch.cuda.stream(stream) if stream is not None else None
    if ctx is not None:
        ctx.__enter__()
    try:
        if plan.reserved.get(key) != nbytes:
            hold = [empty_scratch(nbytes, torch.uint8, dev) for _ in range(ARENAS_IN_FLIGHT)]
            del hold
            plan.reserved[key] = nbytes
        return empty_scratch(nbytes, torch.uint8, dev)
    finally:
        if ctx is not None:
            ctx.__exit__(None, None, None)


_POOLED = {}


def reserve_blocks(tag, nbytes, dev, stream=None, count=16):
    """Park `count` blocks of `nbytes` in the caching allocator's pool of `stream` (once per tag/size).  For the few
    per-step tensors that are used on more than one stream (`record_stream` defers their reuse, so how many are alive at
    once depends on timing): without this the pool occasionally grows by a cudaMalloc in the middle of training, which
    stalls the busy GPU for tens of milliseconds."""
    key = (tag, dev.index, stream.cuda_stream if stream is not None else 0)
    if _POOLED.get(key, 0) >= nbytes:
        return
    ctx = torch.cuda.stream(stream) if stream is not None else None
    if ctx is not None:
        ctx.__enter__()
    try:
        hold = [empty_scratch(nbytes, torch.uint8, dev) for _ in range(count)]
        del hold
    finally:
        if ctx is not None:
            ctx.__exit__(None, None, None)
    _POOLED[key] = nbytes


def _view(arena, ptr, shape, dtype, ld=None):
    """A tensor over arena memory at device address `ptr` that is NOT an autograd view of the arena (Tensor.set_ on the
    shared storage), so it can be returned from an autograd Function and outlive the arena tensor object.  ld: row pitch
    of a 2-D [rows, c] view (> c: a column slice of a wider matrix)."""
    esz = torch.empty(0, dtype=dtype).element_size()
    off = ptr - arena.data_ptr()
    assert off >= 0 and off % esz == 0
    shape = tuple(int(s) for s in shape)
    if ld is None:
        strides, acc = [], 1
        for s in reversed(shape):
            strides.append(acc)
            acc *= s
        strides = tuple(reversed(strides))
    else:
        assert len(shape) == 2 and ld >= shape[1]
        strides = (int(ld), 1)
    n = 1 + sum((s - 1) * st for s, st in zip(shape, strides)) if all(shape) else 0
    assert off + n * esz <= arena.numel()
    t = torch.empty(0, dtype=dtype, device=arena.device)
    t.set_(arena.untyped_storage(), off // esz + arena.storage_offset() // esz, shape, strides)
    return t


class _Run:
    """One forward's record: arena + state blob, enough for the backward call and for queries."""

    def __init__(self, plan, arena, state, precision):
        self.plan, self.arena, self.state, self.precision = plan, arena, state, precision

    def query(self, what, idx):
        out = (ctypes.c_longlong * 8)()
        check(_lib.load().vc_exec_query(self.state.ctypes.data, what, idx, out), 'vc_exec_query')
        return [int(v) for v in out]

    def feature(self, slot):
        p, _, rows, c = self.query(1, slot)[:4]
        return _view(self.arena, p, (rows, c), torch.float32)

    def feature_bf16(self, slot):
        _, pb, rows, c = self.query(1, slot)[:4]
        return _view(self.arena, pb, (rows, c), torch.bfloat16) if pb else None

    def indices(self, iset):
        p, n, ndim, s0, s1, s2 = self.query(2, iset)[:6]
        return _view(self.arena, p, (n, 1 + ndim), torch.int32), [s0, s1, s2][:ndim]

    def deterministic_bytes(self):
        """(deterministic mode or not, arena bytes its partials, tables and operands take in this run so far)."""
        used, det_bytes, det = self.query(0, 0)[:3]
        return bool(det), det_bytes

    def count(self, iset):
        """Static mode: the device int32[1] row count of an index set (a view into the arena, or the StaticSpec's own n_dev
        for the input's rows)."""
        p = self.query(2, iset)[6]
        if p and self.static is not None and p == self.static.n_dev.data_ptr():
            return self.static.n_dev
        return _view(self.arena, p, (1,), torch.int32) if p else None

    def kept_rows(self):
        """The rows each layer discard of this run kept, one int32 tensor per site in site order: [k] in exact mode;
        capacity-sized with a -1 tail and the device count as `.num_rows` in static mode."""
        out = []
        for site, op in sorted(self.plan.discards):
            p, k, pk, n_in, _ = self.query(5, op)[:5]
            t = _view(self.arena, p, (k,), torch.int32)
            if self.static is not None:
                t.num_rows = _view(self.arena, pk, (1,), torch.int32)
            out.append(t)
        return out

    def rulebook(self, rb):
        """(nbr [K, n_out] int32, nbr_bwd or None, pair_num or None, meta dict) — tests compare these with the oracle."""
        p, pbw, ppn, K, n_in, n_out, subm, unique = self.query(3, rb)
        nbr = _view(self.arena, p, (K, n_out), torch.int32)
        nbw = _view(self.arena, pbw, (K, n_in), torch.int32) if pbw else None
        pn = _view(self.arena, ppn, (K,), torch.int32) if ppn else None
        return nbr, nbw, pn, dict(K=K, n_in=n_in, n_out=n_out, subm=bool(subm), unique=bool(unique))

    def _rows_view(self, ptr, rows, c, ld, dtype, iset):
        """[rows, c] view with row pitch ld, None for a null pointer or memory outside the arena; static mode: `rows` is the
        capacity and the view carries the device row count of index set `iset` as `.num_rows`."""
        if not ptr or not (self.arena.data_ptr() <= ptr < self.arena.data_ptr() + self.arena.numel()):
            return None
        t = _view(self.arena, ptr, (rows, c), dtype, ld)
        if self.static is not None:
            t.num_rows = self.static.n_dev if iset == 0 else self.count(iset)
        return t

    def slot(self, slot):
        """Feature slot `slot` as {'f32', 'bf16', 'grad'}: [rows, c] views honouring each buffer's row pitch (a column slice of
        an in-place concat, or of its gradient, has a pitch above c), None where the run keeps no such buffer.  After the
        backward, 'grad' is the slot's final input gradient (None for a published slot no layer reads: its gradient is the
        caller's own tensor).  Static mode: capacity rows, the device row count as `.num_rows`."""
        f32, bf16, rows, c, ld, grad, gld = self.query(1, slot)[:7]
        iset = self.plan.slot_isets()[slot]
        if slot == 0:        # the caller's input features
            x = self.feats
            if self.static is not None:
                x = x.view(x.shape)
                x.num_rows = self.static.n_dev
        return {'f32': x if slot == 0 else self._rows_view(f32, rows, c, ld, torch.float32, iset),
                'bf16': self._rows_view(bf16, rows, c, ld, torch.bfloat16, iset),
                'grad': self._rows_view(grad, rows, c, gld, torch.float32, iset)}

    def layer_forward(self, layer):
        """{'x': the conv's fp32 output [n_out, c_out], 'stats': [4, c_out] = BN scale, shift, mean, invstd, 'rb', 'in_slot',
        'out_slot'} of `layer` (static mode: x with `.num_rows`); its input and output are slot(in_slot) / slot(out_slot)."""
        x, _, stats, _, rb, in_slot, out_slot = self.query(4, layer)[:7]
        n_out, cout = self.query(3, rb)[5], self.plan.layers[layer][0].out_channels
        return {'x': self._rows_view(x, n_out, cout, cout, torch.float32, self.plan.slot_isets()[out_slot]),
                'stats': _view(self.arena, stats, (4, cout), torch.float32), 'rb': rb, 'in_slot': in_slot, 'out_slot': out_slot}

    def layer_backward(self, layer):
        """What the backward used for `layer`: {'dy': upstream gradient (None where it is the caller's own gradient tensor of a
        published slot), 'dx' / 'dxb': the BN backward's fp32 / bf16 output (each None where the run did not write it),
        [n_out, c_out] views, static mode with `.num_rows`} and the kernel
        names it ran ('fwd', 'wgrad', 'dgrad'; 'dgrad' None for a layer without an input gradient).  The gather-form dgrad
        of a many-to-one table reads [dx; S] (fp32) or [dxb; S] (bf16), S the sums of dx over the rows of each pixel at
        its lowest row: 'sums' is that S, else None."""
        dy, dy_ld, dx, dxb, fwd, wgrad, dgrad = self.query(6, layer)[:7]
        rb, out_slot = self.query(4, layer)[4], self.query(4, layer)[6]
        n_out, cout = self.query(3, rb)[5], self.plan.layers[layer][0].out_channels
        iset = self.plan.slot_isets()[out_slot]
        out = {'dy': self._rows_view(dy, n_out, cout, dy_ld, torch.float32, iset),
               'dx': self._rows_view(dx, n_out, cout, cout, torch.float32, iset),
               'dxb': self._rows_view(dxb, n_out, cout, cout, torch.bfloat16, iset),
               'fwd': KIND_NAMES[fwd], 'wgrad': KIND_NAMES[wgrad], 'dgrad': KIND_NAMES.get(dgrad), 'sums': None}
        if out['dgrad'] in ('conv_dgrad_gather2d', 'conv_dgrad_gather2d_tc'):
            tc = out['dgrad'] == 'conv_dgrad_gather2d_tc'
            p, dt = (dxb, torch.bfloat16) if tc else (dx, torch.float32)
            out['sums'] = self._rows_view(p + n_out * cout * (2 if tc else 4), n_out, cout, cout, dt, iset)
        return out


class LazyIndiceDict(dict):
    """`SparseConvTensor.indice_dict` of the tensors a plan publishes: {indice_key: ops.Rulebook} like the module path
    leaves behind (spconv caches its indice pairs there), but materialised on first access — building a dozen tensor
    views per step for a dictionary nobody reads would be pure host overhead.  `group`: the index-set group
    (Plan.iset_group) of the tensors the dictionary belongs to."""

    def __init__(self, run, coords0, shape0, group=0):
        super().__init__()
        self._src = (run, coords0, shape0, group)

    def _fill(self):
        if self._src is None:
            return
        run, coords0, shape0, group = self._src
        self._src = None
        for rb, (keys, ndim, i_in, i_out) in run.plan.rb_keys.items():
            if not keys or run.plan.iset_group[i_out] != group:
                continue
            nbr, nbw, pn, meta = run.rulebook(rb)
            oidx, oshape = (coords0, list(shape0)) if i_out == 0 else run.indices(i_out)
            book = ops.Rulebook(meta['subm'], ndim, meta['K'], meta['n_in'], meta['n_out'], nbr, nbw, pn, oidx, oshape,
                                meta['unique'])
            book._keepalive = run
            for k in keys:
                dict.__setitem__(self, k, book)

    def __getitem__(self, k):
        self._fill()
        return dict.__getitem__(self, k)

    def __contains__(self, k):
        self._fill()
        return dict.__contains__(self, k)

    def __iter__(self):
        self._fill()
        return dict.__iter__(self)

    def __len__(self):
        self._fill()
        return dict.__len__(self)

    def get(self, k, default=None):
        self._fill()
        return dict.get(self, k, default)

    def items(self):
        self._fill()
        return dict.items(self)

    def keys(self):
        self._fill()
        return dict.keys(self)

    def values(self):
        self._fill()
        return dict.values(self)


def _layer_ptrs(plan, grad_base=0):
    """[n_layers, 9] uint64 pointer table of vc_exec_*.  The parameter / buffer columns are cached per plan and re-read
    only when a weight's address changes (module.to(), load of a new tensor object); the gradient columns are
    `grad_base` + fixed offsets into the step's flat gradient buffer."""
    oi, of, lf, sizes, offs = plan.finalize()
    key = tuple((conv.weight.data_ptr(), bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(),
                 bn.running_var.data_ptr(), bn.num_batches_tracked.data_ptr() if bn.num_batches_tracked is not None else 0)
                for conv, bn in plan.layers)
    cached = getattr(plan, '_ptr_cache', None)
    if cached is None or cached[0] != key:
        tab = np.zeros((len(plan.layers), PCOLS), dtype=np.uint64)
        for i, (conv, bn) in enumerate(plan.layers):
            nbt = bn.num_batches_tracked
            tab[i, 0] = conv.weight.data_ptr()
            tab[i, 1] = bn.weight.data_ptr()
            tab[i, 2] = bn.bias.data_ptr()
            tab[i, 3] = bn.running_mean.data_ptr()
            tab[i, 4] = bn.running_var.data_ptr()
            tab[i, 5] = nbt.data_ptr() if nbt is not None else 0
        goff = (4 * offs[:-1].reshape(-1, 3)).astype(np.uint64)
        plan._ptr_cache = cached = (key, tab, goff)
    tab = cached[1].copy()
    if grad_base:
        tab[:, 6:9] = cached[2] + np.uint64(grad_base)
    return tab


class StaticSpec:
    """Static (CUDA-graph capturable) execution of a plan: `n_dev` int32[1] device tensor = number of valid input rows
    (the feature / coordinate tensors passed to the plan are then CAPACITY sized), `caps` {index-set id: row capacity} for
    the strided convs' output sets, `overflow` int32[1] device tensor receiving the largest row count that did not fit."""

    def __init__(self, n_dev, caps, overflow, alias_params=False):
        self.n_dev, self.caps, self.overflow = n_dev, dict(caps), overflow
        self.alias_params = alias_params      # differentiate w.r.t. per-call leaf aliases of the parameters (run_plan)
        self.param_aliases = {}
        # phased execution (graph.PipelinedStep): 1 = only the index operators (run_index), 2 = only the feature operators
        # (run_plan), both in the caller-owned `arena` (deterministic bump allocation: the two phases agree on every address)
        self.phase, self.arena = 0, None
        self._arr = None

    def caps_array(self):
        if self._arr is None:
            a = np.zeros(64, dtype=np.int32)
            for k, v in self.caps.items():
                a[int(k)] = int(v)
            self._arr = a
        return self._arr


def _index_streams(dev, inputs_ready=False):
    """(side, side2) index streams of vc_exec_forward, None to share the previous one.  No side2 (image branch) with
    `inputs_ready`: the index streams then do not wait for main, and the arena is registered with ONE side stream."""
    side = ops.side(dev).stream if TWO_STREAMS else None
    return side, (ops.side2(dev) if (side is not None and THREE_STREAMS and not inputs_ready) else None)


_NO_EXCHANGE = (None, None, _lib.EXCHANGE_FN(), None)     # (a NULL vc_bn_exchange_fn: plain BatchNorm)


class _Exchange:
    """One step's SyncBatchNorm exchange (sync_bn): the float64 slot buffer (Plan.sync_slots; alive from the forward to its
    backward, which reads the forward slots' global counts) and the vc_bn_exchange_fn callback that hands a slot to
    `reducer(slot, (tag, layer, 'forward' | 'backward'))`.  An exception in the reducer fails the C call and is re-raised."""

    def __init__(self, plan, reducer, tag, dev):
        self.off, n = plan.sync_slots()
        self.buf = empty_scratch(max(n, 1), torch.float64, dev)    # (every slot is written before it is reduced)
        self.reducer, self.tag, self.error = reducer, tag, None
        self.fn = _lib.EXCHANGE_FN(self._call)

    def _call(self, user, layer, direction, ptr, n):
        try:
            i = (ptr - self.buf.data_ptr()) // 8
            self.reducer(self.buf[i:i + n], (self.tag, int(layer), 'backward' if direction else 'forward'))
            return 0
        except BaseException as e:      # (an exception must not cross the C frames)
            self.error = e
            return 1

    def args(self):
        return self.buf.data_ptr(), self.off.ctypes.data, self.fn, None

    def raise_error(self):
        if self.error is not None:
            e, self.error = self.error, None
            raise e


def _exec_forward(plan, feats, coords, spatial_shape, batch_size, proj, training, precision, static, arena, side, side2,
                  side_waits_main, seed=None, xchg=None):
    """One vc_exec_forward_sync call (only one phase where static.phase says so) -> (return code, state blob).  seed:
    device int64[1] of the plan's layer discards; xchg: the _Exchange of a SyncBatchNorm step, else None.
    torch.are_deterministic_algorithms_enabled() selects the deterministic mode (flags bit 2), which the state records for
    the backward; a captured graph keeps the mode of its capture."""
    oi, of, lf, _, _ = plan.finalize()
    tab, lib, dev = _layer_ptrs(plan), _lib.load(), feats.device
    state = np.zeros(lib.vc_exec_state_bytes(), dtype=np.uint8)
    rc = lib.vc_exec_forward_sync(
        oi.ctypes.data, of.ctypes.data, oi.shape[0], tab.ctypes.data, lf.ctypes.data, len(plan.layers), feats.data_ptr(),
        feats.shape[1], coords.data_ptr(), feats.shape[0], _lib.host_i32(spatial_shape), int(batch_size),
        proj.data_ptr() if proj is not None else None, int(training), int(precision == 'bf16'),
        1 | (4 if torch.are_deterministic_algorithms_enabled() else 0) | ((static.phase if static is not None else 0) << 8),
        arena.data_ptr(), arena.numel(), _pinned(dev).data_ptr(),
        ops.tc_error_flag(dev).data_ptr(), state.ctypes.data, state.size, ops._stream(),
        side.cuda_stream if side is not None else None, int(side_waits_main),
        static.caps_array().ctypes.data if static is not None else None, static.n_dev.data_ptr() if static is not None else None,
        static.overflow.data_ptr() if static is not None else None, side2.cuda_stream if side2 is not None else None,
        seed.data_ptr() if seed is not None else None, *(xchg.args() if xchg is not None else _NO_EXCHANGE))
    if xchg is not None:
        xchg.raise_error()
    return rc, state


class PlanFn(torch.autograd.Function):
    """forward: (features of the published slots..., ) ; backward: gradients of every layer's weight / gamma / beta."""

    @staticmethod
    def forward(ctx, plan, holder, feats, coords, spatial_shape, batch_size, proj, training, precision, inputs_ready, static,
                with_bwd, seed, xchg, *params):
        ctx.set_materialize_grads(False)     # published tensors the loss does not touch arrive as None, not as zeros
        dev = feats.device
        feats = feats.contiguous()
        n0 = feats.shape[0]
        side_obj, side2_obj = _index_streams(dev, inputs_ready)
        inflight = None
        if static is not None:
            inputs_ready = False             # under capture the side stream must fork from the capturing stream
        else:
            inflight = _throttle(plan, dev)
        for attempt in range(3 if xchg is None else 1):
            # (SyncBatchNorm: no re-run — the exchanges of the failed walk were already enqueued, the other ranks would pair
            #  them with the wrong ones.  So twice the largest arena use per input row seen so far instead of 1.3x; a batch
            #  denser than that still fails, on its rank, and the other ranks wait in their exchanges: DESIGN.md section 6)
            nbytes = _arena_bytes(plan, n0, dev, with_bwd, 1.3 if xchg is None else 2.0)
            if static is not None and static.arena is not None:
                arena = static.arena              # phased execution: the index phase already built its part in there
            elif static is not None:
                # (inside a capture: the graph's own pool.  No record_stream: the side / wgrad streams are forked from and
                #  joined back into the calling stream inside vc_exec_forward / vc_exec_backward, so every later use of the
                #  block in the calling stream's order comes after all of this step's uses)
                arena = empty_scratch(nbytes, torch.uint8, dev)
            elif side_obj is not None:
                # The arena belongs to the SIDE stream (its index kernels are the first writers, possibly while main still
                # runs the previous step); main's uses are registered with record_stream, so the caching allocator recycles
                # the block only after both streams are done with it.
                arena = _alloc_arena(plan, nbytes, dev, side_obj)
                arena.record_stream(torch.cuda.current_stream(dev))
            else:
                arena = _alloc_arena(plan, nbytes, dev, None)
            rc, state = _exec_forward(plan, feats, coords, spatial_shape, batch_size, proj, training, precision, static, arena,
                                      side_obj, side2_obj, side_waits_main=not (inputs_ready and side_obj is not None), seed=seed,
                                      xchg=xchg)
            if rc != VC_ERR_WORKSPACE:
                break
            # too small (first use of a plan on an unusually dense batch): the call is restartable — nothing it enqueued is
            # read by anyone — so take a bigger arena and run it again
            plan.arena_bytes[(dev.index, bool(with_bwd))] = 2 * arena.numel()
        check(rc, 'vc_exec_forward')
        if inflight is not None:
            tail = torch.cuda.Event()
            tail.record()
            inflight.append(tail)
        run = _Run(plan, arena, state, precision)
        run.static, run.n0, run.training, run.with_bwd, run.feats = static, n0, bool(training), bool(with_bwd), feats
        run.xchg = xchg
        holder.append(run)
        if not with_bwd:
            _note_arena_use(plan, dev, False, run.query(0, 0)[0], n0)
        if TIMING:
            global LAST_RUN
            LAST_RUN = run
        ctx.run, ctx.feats, ctx.coords, ctx.proj, ctx.seed = run, feats, coords, proj, seed
        return tuple(run.feature(slot) for _, slot, _ in plan.published)

    @staticmethod
    def backward(ctx, *grads):
        lib = _lib.load()
        run = ctx.run
        plan = run.plan
        oi, of, lf, sizes, offs = plan.finalize()
        dev = run.arena.device
        if run.static is None:
            reserve_blocks(('flat_grad', id(plan)), 4 * int(offs[-1]), dev)
        flat = empty_scratch(int(offs[-1]), torch.float32, dev)     # (every element is written by vc_exec_backward)
        tab = _layer_ptrs(plan, flat.data_ptr())
        gs = [None if g is None else g.contiguous() for g in grads]
        slots = np.array([slot for _, slot, _ in plan.published], dtype=np.int32)
        ext = np.array([0 if g is None else g.data_ptr() for g in gs], dtype=np.uint64)
        ws = _wgrad_stream(dev)
        if ws is not None and run.static is None:
            flat.record_stream(ws)
            run.arena.record_stream(ws)
        xchg = run.xchg
        rc = lib.vc_exec_backward_sync(oi.ctypes.data, of.ctypes.data, oi.shape[0], tab.ctypes.data, lf.ctypes.data,
                                       len(plan.layers), slots.ctypes.data, ext.ctypes.data, len(gs), run.arena.data_ptr(),
                                       run.arena.numel(), ops.tc_error_flag(dev).data_ptr(), run.state.ctypes.data, ops._stream(),
                                       ws.cuda_stream if ws is not None else None,
                                       *(xchg.args() if xchg is not None else _NO_EXCHANGE))
        if xchg is not None:
            xchg.raise_error()
        if rc == VC_ERR_WORKSPACE:
            # (a forward taken without autograd's knowledge of a later backward: the next step's arena is sized for it)
            plan.arena_bytes[(dev.index, run.with_bwd)] = 2 * run.arena.numel()
        check(rc, 'vc_exec_backward')
        _note_arena_use(plan, dev, run.with_bwd, run.query(0, 0)[0], run.n0)
        run.flat_grad = flat
        views = flat.split(sizes)
        out = [v.view_as(p) for v, p in zip(views, plan.params())]
        return (None,) * 14 + tuple(out)


def run_index(plan, feats, coords_i32, spatial_shape, batch_size, proj, training, precision, static, seed=None):
    """Phase 1 of a phased static execution: enqueue ONLY the index operators of the plan (rulebooks, projection) into
    `static.arena`; `run_plan` with `static.phase == 2` later enqueues the feature operators over the same arena."""
    ops._require_cuda(feats, coords_i32)
    assert static is not None and static.arena is not None and static.phase == 1
    rc, _ = _exec_forward(plan, feats, coords_i32, spatial_shape, batch_size, proj, training, precision, static, static.arena,
                          *_index_streams(feats.device), side_waits_main=True, seed=seed)
    check(rc, 'vc_exec_forward (index phase)')


def run_plan(plan, feats, coords_i32, spatial_shape, batch_size, proj, training, precision, inputs_ready=False, static=None,
             seed=None, reducer=None, tag=''):
    """-> (run record, {name: (features, indices, spatial_shape, bf16 shadow, device row count or None)}).  `coords_i32`
    [N,4] int32 contiguous (b,z,y,x).  inputs_ready: the caller vouches that `coords_i32` and `proj` are complete in the
    SIDE stream's order (resident from an earlier step, or produced on / synchronised with ops.side(device).stream): the
    index pipeline then does not wait for the main stream and overlaps the previous step's backward.  static: a StaticSpec
    (capacity-sized tensors, device row counts, no host synchronisation: CUDA-graph capturable).  seed: device int64[1], the
    draw of the plan's layer discards (Plan.discard), read on the index stream after everything queued on main so far.
    reducer (training only): the SyncBatchNorm exchange — `reducer(slot, (tag, layer, 'forward' | 'backward'))` sums a float64
    slot over the ranks on the current stream (sync_bn); None: plain BatchNorm."""
    ops._require_cuda(feats, coords_i32)
    assert coords_i32.dtype == torch.int32 and coords_i32.is_contiguous()
    inputs_ready = inputs_ready and seed is None       # (the seed is drawn on main: the index stream must wait for it)
    holder = []
    # the arena also holds what a backward saves / stages: sized for it whenever autograd will record this call
    with_bwd = bool(training) or (torch.is_grad_enabled() and (feats.requires_grad or any(p.requires_grad for p in plan.params())))
    params = plan.params()
    if static is not None and with_bwd and static.alias_params:
        # Fresh leaf aliases of the parameters (same storage) for this call.  autograd keeps ONE AccumulateGrad node per leaf
        # alive as long as any earlier graph is, and that node remembers the stream it was created on: a node born in an eager
        # step on the legacy default stream makes the engine synchronise that stream with the capturing one — illegal during
        # CUDA-graph capture (cudaErrorStreamCaptureImplicit).  graph.GraphedStep differentiates w.r.t. the aliases.
        aliases = [p.detach().requires_grad_(True) for p in params]
        static.param_aliases = {id(p): a for p, a in zip(params, aliases)}
        params = aliases
    xchg = _Exchange(plan, reducer, tag, feats.device) if (reducer is not None and training) else None
    outs = PlanFn.apply(plan, holder, feats, coords_i32, list(spatial_shape), batch_size, proj, training, precision,
                        bool(inputs_ready), static, with_bwd, seed, xchg, *params)
    run = holder[0]
    res = {}
    for (name, slot, iset), f in zip(plan.published, outs):
        idx, shape = (coords_i32, list(spatial_shape)) if iset == 0 else run.indices(iset)
        cnt = None
        if static is not None:
            cnt = static.n_dev if iset == 0 else run.count(iset)
        res[name] = (f, idx, shape, (lambda slot=slot: run.feature_bf16(slot)), cnt)    # shadow resolved on first use
    return run, res


class RunCounts:
    """What outlives a run record (whose arena goes back to the allocator with the step's tensors): the row count of every
    strided conv's output set, for sizing a StaticSpec.  Read from the run's host-side state blob on first use: every
    exact-mode forward keeps one, and only capacity sizing ever asks."""

    def __init__(self, run):
        self._rows, self._src = ({}, None) if run.static is not None else (None, copy.copy(run))
        if self._src is not None:
            self._src.arena = None           # (the counts are host values: the step's arena need not stay alive for them)

    @property
    def rows(self):
        if self._rows is None:
            run, self._src, self._rows = self._src, None, {}
            for rb, (keys, ndim, i_in, i_out) in run.plan.rb_keys.items():
                if i_out != i_in and i_out != 0:
                    self._rows[i_out] = int(run.query(2, i_out)[1])
        return self._rows


_LAST_RUNS = weakref.WeakKeyDictionary()     # model -> {stream: RunCounts of the most recent exact-mode run of that stream}


def note_last_run(model, run, stream=''):
    """Keep the row counts of an exact-mode run of one of `model`'s plans.  stream: the batch-key suffix of the input stream
    the plan ran on — '' for VirConvL8x and VirConv8x's LiDAR stream, '_mm' for VirConv8x's virtual-point stream — so that
    one exact step sizes the StaticSpec of every stream."""
    if run.static is None:
        _LAST_RUNS.setdefault(model, {})[stream] = RunCounts(run)


def last_run(model, stream=''):
    """RunCounts of the most recent exact-mode run of `model`'s plan on `stream` (see note_last_run), or None."""
    return _LAST_RUNS.get(model, {}).get(stream)


def measured_caps(run, margin=1.3, grain=1024):
    """{index-set id: capacity} for a StaticSpec from an EXACT-mode run of the same plan on a representative batch (a run
    record or the RunCounts `last_run(model)` keeps): the observed row count of every strided conv's output set times
    `margin`, rounded up to `grain` rows."""
    rows = run.rows if isinstance(run, RunCounts) else RunCounts(run).rows
    return {i: (int(n * margin) + grain - 1) // grain * grain for i, n in rows.items()}


def timing_start():
    global TIMING
    TIMING = True
    check(_lib.load().vc_exec_timing(1), 'vc_exec_timing')


def timing_stop():
    """-> list of (kind name, layer, ms)."""
    global TIMING
    lib = _lib.load()
    n_max = 4096
    ms = (ctypes.c_float * n_max)()
    kl = (ctypes.c_int32 * (2 * n_max))()
    n = lib.vc_exec_timing_read(ms, kl, n_max)
    if n < 0:
        check(n, 'vc_exec_timing_read')
    TIMING = False
    check(lib.vc_exec_timing(0), 'vc_exec_timing')
    return [(KIND_NAMES[kl[2 * i]], int(kl[2 * i + 1]), float(ms[i])) for i in range(n)]


def alg_bytes_flops(run, kind, layer):
    """Algorithmic bytes / FLOPs of one timed conv launch (SURVEY §8d; same formulas as ops.py's per-call accounting):
    every input row read once, every output row written once, one (in, out) pair per rulebook entry, the weights."""
    rb_id, in_slot, out_slot = run.query(4, layer)[4:7]
    _, _, pn, meta = run.rulebook(rb_id)
    conv = run.plan.layers[layer][0]
    cin, cout, K = conv.in_channels, conv.out_channels, meta['K']
    n_in, n_out, P = meta['n_in'], meta['n_out'], int(pn.sum().item())
    w = K * cin * cout
    if kind == 'conv_fwd_tc':
        b = n_in * cin * 2 + n_out * cout * 4 + w * 2
    elif kind in ('conv_dgrad_tc', 'conv_dgrad_scatter_tc'):
        b = n_out * cout * 2 + n_in * cin * 4 + w * 2
    elif kind == 'conv_wgrad_tc':
        b = (n_in * cin + n_out * cout) * 2 + w * 4
    else:
        b = (n_in * cin + n_out * cout + w) * 4
    return b + P * 8, 2 * P * cin * cout
