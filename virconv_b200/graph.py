"""Whole training step (backbone forward + loss + backward) as ONE CUDA graph.

The reference drives every step from Python (`tools/train_utils/train_utils.py:27-57`: `model(batch)`, `loss.backward()`):
~200 kernel launches whose enqueue cost can exceed the kernels' run time on the GPU.
The plan executor's static mode (`executor.StaticSpec`, `vc_exec_forward(..., caps, n0_dev, overflow)`) keeps every
data-dependent row count in device memory and sizes every buffer from host-side capacities, so nothing in a step reads a
device value on the host; `GraphedStep` captures such a step once and replays it:

    step = GraphedStep(model, loss_fn, params)          # model: VirConvL8x in train / eval mode, or VirConv8x in train mode
    for batch in loader:
        loss = step(batch)                              # copies the batch into the graph's input buffers, replays
        optimizer.step()                                # parameter .grad tensors are rewritten in place by every replay

Published tensors inside the graph are capacity sized: `t.features` [cap, C] with a zero tail, `t.indices` [cap, 4] with a
-1 tail, `t.num_rows` a device int32[1]; `loss_fn(batch_dict)` must use `num_rows` where the reference uses `shape[0]`.
A batch whose row counts exceed the captured capacities is detected through the executor's overflow flag (read back
asynchronously, one step late) and handled by re-capturing with larger capacities and re-running that batch.

A model with several input streams (`model.static_streams`: VirConv8x with MM has the LiDAR stream '' and the virtual-point
stream '_mm') gets input buffers, an input capacity, a device row count and an overflow flag per stream; the batch keys of a
stream carry its suffix ('voxel_features_mm', 'points_mm', 'virconv_static_mm').

`GraphedForward` (end of the file) does the same for the test-time backbone forward, ROT_NUM transformed copies included.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, executor, ops


class _MaskedMean(torch.autograd.Function):
    """One library kernel each way (vc_masked_mean_f32 / _bwd_f32): the backward writes the contiguous [N, C] gradient the
    plan executor consumes, so nothing downstream has to expand or copy it."""

    @staticmethod
    def forward(ctx, features, num_rows):
        ops._require_cuda(features, num_rows)
        assert features.dtype == torch.float32 and features.dim() == 2, (features.dtype, features.shape)
        assert num_rows is None or (num_rows.dtype == torch.int32 and num_rows.numel() == 1)
        lib = _lib.load()
        x = features.contiguous()
        out = torch.empty((), dtype=torch.float32, device=x.device)
        ws = torch.empty(lib.vc_masked_mean_ws_bytes(), dtype=torch.uint8, device=x.device)
        _lib.check(lib.vc_masked_mean_f32(ops._p(x), x.shape[0], x.shape[1], ops._p(num_rows), ops._p(out), ops._p(ws), ws.numel(),
                                          ops._stream()), 'vc_masked_mean_f32')
        ctx.shape, ctx.num_rows = x.shape, num_rows
        return out

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        g = g.contiguous()
        dx = torch.empty(ctx.shape, dtype=torch.float32, device=g.device)
        _lib.check(lib.vc_masked_mean_bwd_f32(ops._p(g), ctx.shape[0], ctx.shape[1], ops._p(ctx.num_rows), ops._p(dx), ops._stream()),
                   'vc_masked_mean_bwd_f32')
        return dx, None


def masked_mean(t):
    """Mean over the valid rows of a published tensor: static mode (zero tail, device row count `num_rows`) or exact mode
    (every row)."""
    return _MaskedMean.apply(t.features, getattr(t, 'num_rows', None))


class _Stream:
    """The graph's input side of one stream of the model (batch-key suffix `sfx`, position `i` in the step's device row-count
    and overflow vectors): its capacity-sized input buffers and the StaticSpec capacities of its plan."""

    def __init__(self, sfx, i):
        self.sfx, self.i = sfx, i
        self.caps = {}
        self.cap0 = 0             # input rows the buffers hold (voxels)
        self.cap_pts = 0          # with the in-graph voxeliser: input points the point buffer holds
        self.prev_n = 0


class GraphedStep:
    def __init__(self, model, loss_fn, params=None, margin=1.3, grain=1024, warmup=2, check_overflow=True, voxelizer=None):
        """voxelizer: None — batches carry `voxel_features` / `voxel_coords` (what the reference's dataloader + MeanVFE
        deliver); or a dict(point_cloud_range, voxel_size, max_points_per_voxel, max_voxels, vfe_model) — batches carry the
        collated raw `points` [N, 1+C] and the hash-grid voxelisation + VFE (vc_voxelize_mean) run INSIDE the graph.  With a
        two-stream model the batch also carries `points_mm`, voxelised by a second call with the entries `max_voxels_mm`
        (default: `max_voxels`) and `vfe_model_mm` (default: None, the plain mean)."""
        self.model, self.loss_fn = model, loss_fn
        self.vox = dict(voxelizer) if voxelizer is not None else None
        self.params = list(model.parameters()) if params is None else list(params)
        self.dev = self.params[0].device
        self.margin, self.grain, self.warmup = margin, grain, warmup
        self.check_overflow = check_overflow
        self.graph = None
        self.streams = [_Stream(s, i) for i, s in enumerate(getattr(model, 'static_streams', ('',)))]
        self.recaptures = 0
        self.launches_per_replay = 0
        self._pending = []        # (event, pinned slot) of the replays whose overflow flags have not been looked at yet
        self._slot = 0

    @property
    def cap0(self):
        """Input row capacity of the first (for VirConvL8x: the only) stream."""
        return self.streams[0].cap0

    # ------------------------------------------------------------------------------------------------
    def _round(self, n):
        return (int(n * self.margin) + self.grain - 1) // self.grain * self.grain

    def _vox_arg(self, st, key):
        """A voxeliser setting for stream `st`: `key + st.sfx` where the dict has it, else `key` — except the virtual-point
        stream's VFE, which defaults to the plain mean: the reference's MeanVFE applies its MODEL to the LiDAR stream only
        (mean_vfe.py:51-58)."""
        if key + st.sfx in self.vox:
            return self.vox[key + st.sfx]
        if key == 'vfe_model' and st.sfx == '_mm':
            return None
        return self.vox[key]

    def _voxelize(self, st, points, batch_size, static=False):
        v = self.vox
        return ops.voxelize_mean(points, batch_size, v['point_cloud_range'], v['voxel_size'], v['max_points_per_voxel'],
                                 self._vox_arg(st, 'max_voxels'), self._vox_arg(st, 'vfe_model'), static=static)

    def _exact_step(self, batch):
        """One ordinary (exact-shape, host-synchronised) step; also measures the row counts of this batch, per stream."""
        for p in self.params:
            p.grad = None
        bd = dict(batch)
        if self.vox is not None:
            for st in self.streams:
                f, c, _ = self._voxelize(st, batch['points' + st.sfx], int(batch['batch_size']))
                bd.update({'voxel_features' + st.sfx: f, 'voxel_coords' + st.sfx: c})
        out = self.model(bd)
        loss = self.loss_fn(out)
        loss.backward()
        return loss.detach(), [executor.last_run(self.model, st.sfx) for st in self.streams]

    def _make_buffers(self, batch, runs):
        B = int(batch['batch_size'])
        dev = self.params[0].device if self.vox is not None else batch['voxel_features'].device
        for st, run in zip(self.streams, runs):
            for k, v in executor.measured_caps(run, self.margin, self.grain).items():
                st.caps[k] = max(st.caps.get(k, 0), v)
            if self.vox is not None:
                pts = batch['points' + st.sfx]
                st.cap_pts = max(st.cap_pts, self._round(pts.shape[0]))
                # unused tail rows: last sample's batch index, coordinates far outside the range (dropped by the voxeliser)
                row = torch.zeros(pts.shape[1], dtype=torch.float32)
                row[0] = B - 1
                row[1:4] = -1.0e6
                st.sentinel = row.to(dev)
                st.pts = st.sentinel.repeat(st.cap_pts, 1).contiguous()
                st.prev_n = 0
                st.cap0 = B * int(self._vox_arg(st, 'max_voxels'))
            else:
                vf, vc = batch['voxel_features' + st.sfx], batch['voxel_coords' + st.sfx]
                st.cap0 = max(st.cap0, self._round(vf.shape[0]))
                st.vf = torch.zeros((st.cap0, vf.shape[1]), dtype=torch.float32, device=dev)
                st.vc = torch.full((st.cap0, vc.shape[1]), -1, dtype=vc.dtype, device=dev)
        ns = len(self.streams)
        self.dev, self.B = dev, B
        self.n_dev = torch.zeros(ns, dtype=torch.int32, device=dev)        # input rows of each stream
        self.overflow = torch.zeros(ns, dtype=torch.int32, device=dev)     # each stream's StaticSpec overflow flag
        self.proj = torch.zeros((B, 28), dtype=torch.float32, device=dev)
        # pinned staging for the small per-step host values: a ring of slots, each guarded by an event recorded after its
        # upload — the host runs several replays ahead of the GPU, and rewriting ONE pinned buffer before the previous
        # step's asynchronous copy has executed would hand that step the next step's row counts / projection
        self.STAGE_SLOTS = 8
        self.proj_host = torch.zeros((self.STAGE_SLOTS, B, 28), dtype=torch.float32).pin_memory()
        self.n_host = torch.zeros((self.STAGE_SLOTS, ns), dtype=torch.int32).pin_memory()
        self._stage_ev = [None] * self.STAGE_SLOTS
        self._stage = 0
        self.ovf_host = torch.zeros((8, ns), dtype=torch.int32).pin_memory()
        self.err_host = torch.zeros(8, dtype=torch.int32).pin_memory()
        self._pending, self._slot = [], 0
        for st in self.streams:
            st.spec = executor.StaticSpec(self.n_dev[st.i:st.i + 1], st.caps, self.overflow[st.i:st.i + 1], alias_params=True)

    def _load(self, batch):
        """Copy one batch into the graph's input buffers (asynchronous, current stream).  False (nothing copied) when a
        stream's input does not fit."""
        key = 'points' if self.vox is not None else 'voxel_features'
        ns = [batch[key + st.sfx].shape[0] for st in self.streams]
        if any(n > (st.cap_pts if self.vox is not None else st.cap0) for st, n in zip(self.streams, ns)):
            return False
        if self.vox is not None:
            for st, n in zip(self.streams, ns):
                st.pts[:n].copy_(batch['points' + st.sfx], non_blocking=True)
                if st.prev_n > n:                      # rows of the previous (larger) batch still sit behind this one
                    st.pts[n:st.prev_n] = st.sentinel
                st.prev_n = n
        slot = self._stage
        self._stage = (slot + 1) % self.STAGE_SLOTS
        if self._stage_ev[slot] is not None:
            self._stage_ev[slot].synchronize()         # (8 steps back: has long completed unless the GPU is far behind)
        if self.vox is None:
            for st, n in zip(self.streams, ns):
                st.vf[:n].copy_(batch['voxel_features' + st.sfx], non_blocking=True)
                st.vc[:n].copy_(batch['voxel_coords' + st.sfx], non_blocking=True)
                self.n_host[slot, st.i] = n
            self.n_dev.copy_(self.n_host[slot], non_blocking=True)
        trans = batch.get('aug_param')
        self.proj_host[slot].copy_(torch.from_numpy(ops.projection_params_host(batch['calib'], trans, self.B)))
        self.proj.copy_(self.proj_host[slot], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._stage_ev[slot] = ev
        return True

    def _static_batch(self, batch):
        drop = {k + st.sfx for st in self.streams for k in ('voxel_features', 'voxel_coords', 'points')}
        bd = {k: v for k, v in batch.items() if k not in drop}
        specs = []
        for st in self.streams:
            if self.vox is not None:
                f, c, num, n_dev = self._voxelize(st, st.pts, self.B, static=True)
                spec = executor.StaticSpec(n_dev, st.caps, self.overflow[st.i:st.i + 1], alias_params=True)
                bd.update({'voxel_features' + st.sfx: f, 'voxel_coords' + st.sfx: c, 'voxel_num_points' + st.sfx: num})
            else:
                spec = st.spec
                bd.update({'voxel_features' + st.sfx: st.vf, 'voxel_coords' + st.sfx: st.vc})
            bd['virconv_static' + st.sfx] = spec
            specs.append(spec)
        bd['virconv_proj'] = self.proj
        self._cur_specs = specs
        return bd

    def _static_step(self, batch):
        out = self.model(self._static_batch(batch))
        loss = self.loss_fn(out)
        # torch.autograd.grad w.r.t. the per-call leaf aliases the executor made of the parameters (executor.run_plan): no
        # long-lived AccumulateGrad node (which remembers the stream it was created on) takes part in a captured backward
        alias = {}
        for spec in self._cur_specs:
            alias.update(spec.param_aliases)
        grads = torch.autograd.grad(loss, [alias.get(id(p), p) for p in self.params], allow_unused=True)
        for p, g in zip(self.params, grads):
            p.grad = g
        return loss.detach()

    def _capture(self, batch):
        torch.cuda.synchronize(self.dev)
        loss_e, runs = self._exact_step(batch)
        assert all(r is not None for r in runs), 'GraphedStep needs a backbone running each stream through the plan executor'
        self._make_buffers(batch, runs)
        assert self._load(batch)
        # warm-up of the static path on a side stream (allocator pools, lazy kernel attributes), as torch.cuda.graphs asks for
        s = torch.cuda.Stream(device=self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s):
            for _ in range(max(self.warmup, 1)):
                for p in self.params:
                    p.grad = None
                self._static_step(batch)
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        for p in self.params:
            p.grad = None
        self.overflow.zero_()
        self.graph = torch.cuda.CUDAGraph()
        lib = _lib.load()
        l0 = lib.vc_launch_count()
        with torch.cuda.graph(self.graph):
            self.loss = self._static_step(batch)
        self.launches_per_replay = int(lib.vc_launch_count() - l0)     # this library's kernels inside one replay
        self.recaptures += 1
        torch.cuda.synchronize(self.dev)

    # ------------------------------------------------------------------------------------------------
    def _overflowed(self):
        """Largest overflow reported by the replays that have COMPLETED so far, over all streams (never blocks: the flags of
        a step are read back asynchronously and looked at when its event has fired, typically one or two calls later)."""
        worst = 0
        while self._pending and self._pending[0][0].query():
            ev, slot = self._pending.pop(0)
            worst = max(worst, int(self.ovf_host[slot].max()))
            if int(self.err_host[slot]) != 0:
                raise _lib.VirConvLibraryError('a tensor-core kernel\'s pipeline wait timed out inside a replayed step '
                                               '(error flag set): the results of that step are invalid')
        return worst

    def __call__(self, batch):
        """-> the step's loss (a device tensor owned by the graph: read or copy it before the next call)."""
        if self.graph is None:
            self._capture(batch)
        if self.check_overflow and self._overflowed():
            # an EARLIER batch did not fit: its gradients were computed on clamped row sets.  Grow and re-capture; the
            # caller sees the event through `recaptures` (a training loop may want to discard those optimizer steps).
            self.margin *= 1.25
            self._capture(batch)
        if not self._load(batch):
            self.margin *= 1.25
            self._capture(batch)            # more input rows than the input buffers hold
            assert self._load(batch)
        self.graph.replay()
        if self.check_overflow:
            if len(self._pending) >= self.ovf_host.shape[0]:    # (host far ahead of the GPU: wait for the oldest read-back)
                self._pending[0][0].synchronize()
                if self._overflowed():
                    self.margin *= 1.25
                    self._capture(batch)
                    return self(batch)
            slot = self._slot
            self._slot = (slot + 1) % self.ovf_host.shape[0]
            self.ovf_host[slot].copy_(self.overflow, non_blocking=True)
            self.err_host[slot:slot + 1].copy_(ops.tc_error_flag(self.dev), non_blocking=True)
            self.overflow.zero_()
            ev = torch.cuda.Event()
            ev.record()
            self._pending.append((ev, slot))
        return self.loss


class _PipeInstance(GraphedStep):
    """One of the two buffer sets of a PipelinedStep: the step captured as TWO graphs over one caller-owned arena — the index
    graph (voxeliser, rulebooks, projections: everything that depends on coordinates only) and the feature graph (weight images,
    conv + BN + ReLU, loss, backward)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.g_idx = self.g_feat = None
        self.feat_done = None
        self.grads = None

    def _static_batch(self, batch):
        bd = super()._static_batch(batch)
        spec = bd['virconv_static']
        spec.phase, spec.arena = 0, None            # (the spec object is shared between calls when there is no voxeliser)
        return bd

    def _index_part(self, batch):
        bd = self._static_batch(batch)              # (in-graph voxeliser, if any)
        spec = bd['virconv_static']
        spec.phase, spec.arena = 1, self.arena
        self.model.index_phase(bd)
        return bd

    def _feature_part(self, bd):
        spec = bd['virconv_static']
        spec.phase = 2
        out = self.model(bd)
        loss = self.loss_fn(out)
        alias = spec.param_aliases
        grads = torch.autograd.grad(loss, [alias.get(id(p), p) for p in self.params], allow_unused=True)
        self.grads = list(grads)
        return loss.detach()

    def _capture(self, batch):
        torch.cuda.synchronize(self.dev)
        loss_e, runs = self._exact_step(batch)
        assert all(r is not None for r in runs), 'PipelinedStep needs a backbone running through the plan executor'
        self._make_buffers(batch, runs)
        assert self._load(batch)
        s = torch.cuda.Stream(device=self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s):
            for _ in range(max(self.warmup, 1)):        # unphased static steps: allocator pools, kernel attributes, arena size
                for p in self.params:
                    p.grad = None
                self._static_step(batch)
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        plan = self.model._plan()
        self.arena = executor.empty_scratch(executor._arena_bytes(plan, self.cap0, self.dev, True), torch.uint8, self.dev)
        for p in self.params:
            p.grad = None
        self.overflow.zero_()
        lib = _lib.load()
        l0 = lib.vc_launch_count()
        self.g_idx = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_idx):
            self._bd = self._index_part(batch)
        self.g_feat = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_feat):
            self.loss = self._feature_part(self._bd)
        self.launches_per_replay = int(lib.vc_launch_count() - l0)
        self.recaptures += 1
        self.feat_done = None
        torch.cuda.synchronize(self.dev)


class PipelinedStep:
    """GraphedStep with the index work of step t+1 running BESIDE the feature work of step t.

    Consecutive replays of one monolithic graph cannot overlap, so the head of every step — voxelisation, the first rulebook,
    the strided convs' count -> indices -> tables chain — sits exposed in front of its first convolution (the exact-mode executor
    hides it behind the previous step's backward: 2.86 vs 3.01 ms per step).  Here every step is two graphs (see _PipeInstance)
    and there are two buffer sets, used alternately: the index graph of a step is launched on its own stream as soon as ITS
    buffer set is free (two steps back), the feature graph on the caller's stream once the index graph is done.  Rulebooks do not
    depend on the weights, so the overlap does not change what a training step computes.  Parameter `.grad` tensors are switched
    to the buffer set of the step that just ran."""

    def __init__(self, model, loss_fn, params=None, **kwargs):
        streams = tuple(getattr(model, 'static_streams', ('',)))
        if streams != ('',):
            raise ValueError('PipelinedStep phases a one-stream backbone (VirConvL8x); %s has the input streams %s, which have '
                             'no phased form: use GraphedStep' % (type(model).__name__, streams))
        self.inst = [_PipeInstance(model, loss_fn, params, **kwargs) for _ in range(2)]
        self.params = self.inst[0].params
        self.dev = self.inst[0].dev
        self.s_idx = torch.cuda.Stream(device=self.dev)
        self.t = 0

    @property
    def recaptures(self):
        return sum(i.recaptures for i in self.inst)

    @property
    def launches_per_replay(self):
        return self.inst[0].launches_per_replay

    def __call__(self, batch):
        inst = self.inst[self.t & 1]
        self.t += 1
        main = torch.cuda.current_stream(self.dev)
        if inst.g_feat is None:
            inst._capture(batch)
        if inst.check_overflow and inst._overflowed():
            inst.margin *= 1.25
            inst._capture(batch)
        with torch.cuda.stream(self.s_idx):
            if inst.feat_done is not None:
                self.s_idx.wait_event(inst.feat_done)          # the buffer set's previous step (two steps back) is through
            else:
                self.s_idx.wait_stream(main)
            ok = inst._load(batch)
            if ok:
                inst.g_idx.replay()
                ev = torch.cuda.Event()
                ev.record(self.s_idx)
        if not ok:                                             # more input rows than the buffers hold: grow, re-capture, run again
            inst.margin *= 1.25
            inst._capture(batch)
            self.t -= 1
            return self(batch)
        main.wait_event(ev)
        inst.g_feat.replay()
        for p, g in zip(self.params, inst.grads):
            p.grad = g
        if inst.check_overflow:
            if len(inst._pending) >= inst.ovf_host.shape[0]:
                inst._pending[0][0].synchronize()
            slot = inst._slot
            inst._slot = (slot + 1) % inst.ovf_host.shape[0]
            inst.ovf_host[slot].copy_(inst.overflow, non_blocking=True)
            inst.err_host[slot:slot + 1].copy_(ops.tc_error_flag(self.dev), non_blocking=True)
            inst.overflow.zero_()
            e2 = torch.cuda.Event()
            e2.record()
            inst._pending.append((e2, slot))
        inst.feat_done = torch.cuda.Event()
        inst.feat_done.record(main)
        return inst.loss


class GraphedForward:
    """The test-time backbone forward as ONE CUDA graph: VirConvL8x (one copy) or VirConv8x over R = 1..4 transformed copies
    (X_TRANS, ROT_NUM; the batch keys carry the reference's suffixes '', '1', '2', ...), with the model in eval mode.

        fwd = GraphedForward(model.eval())                 # voxelised batches; voxelizer=dict(...) takes the collated points
        for batch in loader:
            out = fwd(batch)                               # copies the batch into the graph's input buffers, replays once

    VirConv8x runs its static eval forward (backbone.EvalStaticSpec): vc_xbatch_pack of the R LiDAR copies, the LiDAR plan
    over the [D, H, 4W] grid, vc_xbatch_split of x_conv3 / x_conv4 / out, and one static run of the virtual-point plan per
    copy — no host read of any row count.  The exact eager eval forward reads four strided-conv row counts per plan call and
    one torch.nonzero per split tensor and copy.  Everything runs under torch.no_grad(): nothing is saved for a backward.

    The returned dict is the batch plus the published keys of the eager eval forward, with the static contract: capacity-sized
    features with a zero tail, indices with a -1 tail, the device int32 row count `.num_rows` (SparseConvTensor.dense() and
    ops.voxel2pinds use it).  Its tensors belong to the graph and are valid until the next call.  bev=True also runs
    HeightCompression (height_compression.py:15-36) in the graph: 'spatial_features{i}' [B, C*D, H, W] and
    'spatial_features_stride{i}' per copy.

    Capacities: every plan of every copy gets its own StaticSpec, sized from one exact eval forward of the first batch (times
    `margin`), and its own overflow flag.  check_overflow='sync' (default): each call reads this replay's overflow and error
    flags before returning; a batch that did not fit is re-run after a re-capture with larger capacities, so a returned
    result never comes from clamped row sets.  'async': the flags are read one call late, as GraphedStep does (the result of
    an overflowing batch is then returned, and `recaptures` grows on the next call).

    voxelizer: as GraphedStep's — the batch then carries 'points{i}' (and 'points_mm{i}' for VirConv8x with MM) instead of the
    voxel keys, and vc_voxelize_mean runs inside the graph once per stream and copy; the virtual-point stream's settings are
    the '_mm' entries ('max_voxels_mm', 'vfe_model_mm', default the plain mean)."""

    STAGE_SLOTS = 8

    def __init__(self, model, margin=1.3, voxelizer=None, bev=False, check_overflow='sync', grain=1024, warmup=2):
        from .backbone import VirConv8x, VirConvL8x
        if not isinstance(model, (VirConv8x, VirConvL8x)):
            raise ValueError('GraphedForward captures a VirConvL8x or VirConv8x backbone, got %s' % type(model).__name__)
        if model.training:
            raise ValueError('GraphedForward captures the test-time forward: call model.eval() first (a captured training step '
                             'is graph.GraphedStep)')
        if check_overflow not in ('sync', 'async'):
            raise ValueError("check_overflow: 'sync' or 'async', got %r" % (check_overflow,))
        self.model = model
        self.x_batched = isinstance(model, VirConv8x)
        self.mm = self.x_batched and model.mm
        self.vox = dict(voxelizer) if voxelizer is not None else None
        self.margin, self.grain, self.warmup, self.bev, self.check_overflow = margin, grain, warmup, bool(bev), check_overflow
        self.dev = next(model.parameters()).device
        self.graph, self.R = None, None
        self.recaptures = 0
        self.launches_per_replay = 0
        self.overflow_events = []         # {plan key: rows that did not fit} of every replay that overflowed
        self._pending, self._slot = [], 0

    # -- the copies of a batch and their streams ------------------------------------------------------------------
    @staticmethod
    def _sfx(R):
        return [''] + [str(i) for i in range(1, R)]

    def input_streams(self, R):
        """Batch-key suffixes of the input streams of an R-copy forward: the LiDAR copies '', '1', ... then (MM) the virtual-
        point copies '_mm', '_mm1', ..."""
        sfx = self._sfx(R)
        return sfx + (['_mm' + s for s in sfx] if self.mm else [])

    def plan_streams(self, R):
        """Keys (executor.last_run) of the plan runs of an R-copy forward, one StaticSpec and overflow flag each: '' = the
        x-batched LiDAR plan (VirConvL8x: its only plan), '_mm{i}' = the virtual-point plan of copy i."""
        return [''] + (['_mm' + s for s in self._sfx(R)] if self.mm else [])

    def copies(self, batch):
        """R, the number of transformed copies of `batch` (transform_param [B, R, 3]; 1 without it), after the refusals."""
        R = int(batch['transform_param'].shape[1]) if batch.get('transform_param') is not None else 1
        if not self.x_batched and R != 1:
            raise ValueError('GraphedForward: VirConvL8x runs one copy (VirConv-L.yaml sets no X_TRANS); transform_param has '
                             '%d' % R)
        if not 1 <= R <= ops.XBATCH_MAX:
            raise ValueError('GraphedForward: VirConv8x batches 1..%d transformed copies along x (the factor 4 of the '
                             '[D, H, 4W] grid is fixed, spconv_backbone.py:360); transform_param has %d' % (ops.XBATCH_MAX, R))
        keys = (['points'] if self.vox is not None else ['voxel_features', 'voxel_coords'])
        missing = [k + s for s in self.input_streams(R) for k in keys if batch.get(k + s) is None]
        if missing:
            raise ValueError('GraphedForward: the batch has no %s' % ', '.join(missing))
        return R

    def _vox_arg(self, st, key):
        """A voxeliser setting for input stream `st` ('_mm...' streams: the '_mm' entry where given; their VFE defaults to the
        plain mean, as GraphedStep's)."""
        if st.sfx.startswith('_mm'):
            if key + '_mm' in self.vox:
                return self.vox[key + '_mm']
            if key == 'vfe_model':
                return None
        return self.vox[key]

    def _voxelize(self, st, points, batch_size, static=False):
        v = self.vox
        return ops.voxelize_mean(points, batch_size, v['point_cloud_range'], v['voxel_size'], v['max_points_per_voxel'],
                                 self._vox_arg(st, 'max_voxels'), self._vox_arg(st, 'vfe_model'), static=static)

    def _round(self, n):
        return (int(n * self.margin) + self.grain - 1) // self.grain * self.grain

    def _bev(self, out):
        """HeightCompression (height_compression.py:15-36) of every copy."""
        for s in self._sfx(self.R):
            t = out['encoded_spconv_tensor' + s]
            d = t.dense()
            n, c, dd, h, w = d.shape
            out['spatial_features' + s] = d.view(n, c * dd, h, w)
            out['spatial_features_stride' + s] = out['encoded_spconv_tensor_stride' + s]
        return out

    # -- capture ---------------------------------------------------------------------------------------------------
    def _exact(self, batch):
        """One exact eager eval forward (host-synchronised): measures every plan's row counts."""
        executor._LAST_RUNS.pop(self.model, None)
        bd = dict(batch)
        B = int(batch['batch_size'])
        with torch.no_grad():
            if self.vox is not None:
                for st in self.streams:
                    f, c, _ = self._voxelize(st, batch['points' + st.sfx], B)
                    bd.update({'voxel_features' + st.sfx: f, 'voxel_coords' + st.sfx: c})
            self.model(bd)
        runs = [executor.last_run(self.model, k) for k in self.plan_keys]
        if any(r is None for r in runs):
            from .backbone import _module_path_reason
            st = self.streams[0]
            raise ValueError('GraphedForward: the eval forward does not run through the plan executor (%s)'
                             % _module_path_reason(bd['voxel_features' + st.sfx]))
        return runs

    def _make_buffers(self, batch, runs):
        B = int(batch['batch_size'])
        self.B = B
        self.caps = {}
        for k, run in zip(self.plan_keys, runs):
            self.caps[k] = executor.measured_caps(run, self.margin, self.grain)
        for st in self.streams:
            if self.vox is not None:
                pts = batch['points' + st.sfx]
                st.cap_pts = self._round(pts.shape[0])
                row = torch.zeros(pts.shape[1], dtype=torch.float32)
                row[0] = B - 1
                row[1:4] = -1.0e6             # out of range: the voxeliser drops the unused tail rows
                st.sentinel = row.to(self.dev)
                st.pts = st.sentinel.repeat(st.cap_pts, 1).contiguous()
                st.cap0 = B * int(self._vox_arg(st, 'max_voxels'))
            else:
                vf = batch['voxel_features' + st.sfx]
                st.cap0 = self._round(vf.shape[0])
                st.vf = torch.zeros((st.cap0, vf.shape[1]), dtype=torch.float32, device=self.dev)
                st.vc = torch.full((st.cap0, 4), -1, dtype=torch.int32, device=self.dev)
            st.prev_n = 0
        ns = len(self.streams)
        self.n_dev = torch.zeros(ns + 1, dtype=torch.int32, device=self.dev)       # input rows per stream; [-1]: packed LiDAR rows
        self.overflow = torch.zeros(len(self.plan_keys), dtype=torch.int32, device=self.dev)
        self.proj = torch.zeros((self.R, B, 28), dtype=torch.float32, device=self.dev)
        S = self.STAGE_SLOTS
        self.proj_host = torch.zeros((S, self.R, B, 28), dtype=torch.float32).pin_memory()
        self.n_host = torch.zeros((S, ns + 1), dtype=torch.int32).pin_memory()
        self._stage_ev, self._stage = [None] * S, 0
        self.ovf_host = torch.zeros((8, len(self.plan_keys)), dtype=torch.int32).pin_memory()
        self.err_host = torch.zeros(8, dtype=torch.int32).pin_memory()
        self._pending, self._slot = [], 0

    def _load(self, batch):
        """Copy one batch into the input buffers (asynchronous, current stream); False (nothing copied) when a stream does not
        fit.  Rows a larger earlier batch left behind are reset to the tail values, so published input-set tensors keep
        their zero / -1 tails."""
        key = 'points' if self.vox is not None else 'voxel_features'
        ns = [batch[key + st.sfx].shape[0] for st in self.streams]
        if any(n > (st.cap_pts if self.vox is not None else st.cap0) for st, n in zip(self.streams, ns)):
            return False
        slot = self._stage
        self._stage = (slot + 1) % self.STAGE_SLOTS
        if self._stage_ev[slot] is not None:
            self._stage_ev[slot].synchronize()
        for st, n in zip(self.streams, ns):
            if self.vox is not None:
                st.pts[:n].copy_(batch['points' + st.sfx], non_blocking=True)
                if st.prev_n > n:
                    st.pts[n:st.prev_n] = st.sentinel
            else:
                st.vf[:n].copy_(batch['voxel_features' + st.sfx], non_blocking=True)
                st.vc[:n].copy_(batch['voxel_coords' + st.sfx], non_blocking=True)
                if st.prev_n > n:
                    st.vf[n:st.prev_n] = 0
                    st.vc[n:st.prev_n] = -1
                self.n_host[slot, st.i] = n
            st.prev_n = n
        if self.vox is None:
            self.n_dev.copy_(self.n_host[slot], non_blocking=True)
        tp = batch.get('transform_param')
        for i in range(self.R):
            trans = tp[:, i, :] if tp is not None else batch.get('aug_param')
            self.proj_host[slot, i].copy_(torch.from_numpy(ops.projection_params_host(batch['calib'], trans, self.B)))
        self.proj.copy_(self.proj_host[slot], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._stage_ev[slot] = ev
        return True

    def _static_forward(self, batch):
        from .backbone import EvalStaticSpec
        drop = {k + st.sfx for st in self.streams for k in ('voxel_features', 'voxel_coords', 'points')}
        bd = {k: v for k, v in batch.items() if k not in drop}
        counts = {}
        for st in self.streams:
            if self.vox is not None:
                f, c, num, n = self._voxelize(st, st.pts, self.B, static=True)
                bd['voxel_num_points' + st.sfx] = num
            else:
                f, c, n = st.vf, st.vc, self.n_dev[st.i:st.i + 1]
            bd.update({'voxel_features' + st.sfx: f, 'voxel_coords' + st.sfx: c})
            counts[st.sfx] = n
        ovf = {k: self.overflow[j:j + 1] for j, k in enumerate(self.plan_keys)}
        if self.x_batched:
            sfx = self._sfx(self.R)
            lidar = executor.StaticSpec(self.n_dev[-1:], self.caps[''], ovf[''])
            mm = [executor.StaticSpec(counts['_mm' + s], self.caps['_mm' + s], ovf['_mm' + s]) for s in sfx] if self.mm else []
            bd['virconv_eval_static'] = EvalStaticSpec(lidar, [counts[s] for s in sfx], mm, self.proj)
        else:
            bd['virconv_static'] = executor.StaticSpec(counts[''], self.caps[''], ovf[''])
            bd['virconv_proj'] = self.proj[0]
        before = set(bd)
        out = self.model(bd)
        if self.bev:
            self._bev(out)
        self._published = [k for k in out if k not in before]
        return out

    def _capture(self, batch, R):
        torch.cuda.synchronize(self.dev)
        self.R = R
        self.streams = [_Stream(s, i) for i, s in enumerate(self.input_streams(R))]
        self.plan_keys = self.plan_streams(R)
        runs = self._exact(batch)
        self._make_buffers(batch, runs)
        assert self._load(batch)
        s = torch.cuda.Stream(device=self.dev)          # warm-up of the static path (allocator pools, arena sizes)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s), torch.no_grad():
            for _ in range(max(self.warmup, 1)):
                self._static_forward(batch)
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        self.overflow.zero_()
        self.graph = None
        graph = torch.cuda.CUDAGraph()
        lib = _lib.load()
        l0 = lib.vc_launch_count()
        with torch.no_grad(), torch.cuda.graph(graph):
            self.out = self._static_forward(batch)
        self.graph = graph
        self.launches_per_replay = int(lib.vc_launch_count() - l0)
        self.recaptures += 1
        torch.cuda.synchronize(self.dev)

    # -- replay ----------------------------------------------------------------------------------------------------
    def _flags_to_host(self):
        slot = self._slot
        self._slot = (slot + 1) % self.ovf_host.shape[0]
        self.ovf_host[slot].copy_(self.overflow, non_blocking=True)
        self.err_host[slot:slot + 1].copy_(ops.tc_error_flag(self.dev), non_blocking=True)
        self.overflow.zero_()
        ev = torch.cuda.Event()
        ev.record()
        return ev, slot

    def _flag_values(self, slot):
        """-> the largest row count of one replay that did not fit (0: none); a non-zero one is also recorded in
        `overflow_events` as {plan key: rows}."""
        if int(self.err_host[slot]) != 0:
            raise _lib.VirConvLibraryError("a tensor-core kernel's pipeline wait timed out inside a replayed forward (error flag "
                                           "set): the results of that forward are invalid")
        vals = [int(v) for v in self.ovf_host[slot]]
        if max(vals):
            self.overflow_events.append({k: v for k, v in zip(self.plan_keys, vals) if v})
        return max(vals)

    def _overflowed(self):
        """'async': the largest overflow of the replays that have completed so far (never blocks)."""
        worst = 0
        while self._pending and self._pending[0][0].query():
            worst = max(worst, self._flag_values(self._pending.pop(0)[1]))
        return worst

    def _grow(self, batch, R):
        self.margin *= 1.25
        self._capture(batch, R)

    def __call__(self, batch):
        """-> the batch dict plus the published tensors of this forward (owned by the graph: valid until the next call)."""
        R = self.copies(batch)
        if self.graph is None or R != self.R or int(batch['batch_size']) != self.B:
            self._capture(batch, R)
        if self.check_overflow == 'async' and self._overflowed():
            self._grow(batch, R)           # an EARLIER batch did not fit: its result came from clamped row sets
        while True:
            if not self._load(batch):
                self._grow(batch, R)       # more input rows than the buffers hold
                continue
            self.graph.replay()
            if self.check_overflow == 'sync':
                ev, slot = self._flags_to_host()
                ev.synchronize()
                if self._flag_values(slot):
                    self._grow(batch, R)   # this batch did not fit: re-capture and run it again
                    continue
            else:
                if len(self._pending) >= self.ovf_host.shape[0]:
                    self._pending[0][0].synchronize()
                self._pending.append(self._flags_to_host())
            break
        res = dict(batch)
        res.update({k: self.out[k] for k in self._published})
        return res
