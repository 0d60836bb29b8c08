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

or, with the update inside the graph (optim.FusedAdamOneCycle; clipping, weight decay and Adam in two more launches):

    step = GraphedStep(model, loss_fn, optimizer=opt, max_grad_norm=10.0)
    for it, batch in enumerate(loader):
        scheduler.step(it)                              # sets opt.lr / opt.mom; staged to the device by the next call
        loss = step(batch)

Published tensors inside the graph are capacity sized: `t.features` [cap, C] with a zero tail, `t.indices` [cap, 4] with a
-1 tail, `t.num_rows` a device int32[1]; `loss_fn(batch_dict)` must use `num_rows` where the reference uses `shape[0]`.
A batch whose row counts exceed the captured capacities is detected through the executor's overflow flag (read back
asynchronously, one step late) and handled by re-capturing with larger capacities and re-running that batch.

A model with several input streams (`model.static_streams`: VirConv8x with MM has the LiDAR stream '' and the virtual-point
stream '_mm') gets input buffers, an input capacity, a device row count and an overflow flag per stream; the batch keys of a
stream carry its suffix ('voxel_features_mm', 'points_mm', 'virconv_static_mm').

`PipelinedStep` runs the same step as two graphs over two buffer sets, and `GraphedForward` (end of the file) the test-time
backbone forward, ROT_NUM transformed copies included.  All three share one core (`_Captured`): the input buffers and their
loader (`_Inputs`), the capture sequence, and the read-back ring of the overflow and error flags (`_Flags`); each keeps its own
static body and its own reaction to an overflow.
"""
from __future__ import annotations

import gc

import torch

from . import _lib, executor, ops, preprocess, sync_bn


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


def _round(n, margin, grain):
    return (int(n * margin) + grain - 1) // grain * grain


class _Stream:
    """One input stream of a captured model (batch-key suffix `sfx`, position `i` in the device row-count vector) and its
    capacity-sized input buffers: fp32 features `vf` [cap0, C] with a zero tail and int32 coordinates `vc` [cap0, 4] with a
    -1 tail, or, with the in-graph voxeliser, the points `pts` [cap_pts, 1+C] with a `sentinel` tail."""

    def __init__(self, sfx, i):
        self.sfx, self.i = sfx, i
        self.cap0 = 0             # input rows the plan sees (voxels)
        self.cap_pts = 0          # with the in-graph voxeliser: input points the point buffer holds
        self.prev_n = 0           # input rows of the last batch loaded


class _Inputs:
    """The input side of a captured graph: the buffers of every stream, the device row counts `n_dev` (one per stream, then
    `extra_counts` more that the graph itself writes), the device projection blocks `proj` [copies, B, 28], and the pinned
    staging ring the small per-call host values go through.  vox: the voxeliser dict or None; vox_arg(stream, key): its
    setting for one stream (_Captured._vox_arg)."""

    SLOTS = 8

    def __init__(self, sfxs, vox, vox_arg, copies=1, extra_counts=0):
        self.streams = [_Stream(s, i) for i, s in enumerate(sfxs)]
        self.vox, self.vox_arg, self.copies, self.extra_counts = vox, vox_arg, copies, extra_counts
        self.B = None
        # the voxeliser dict's `input_discard` entry, dict(rate=0.8, later_fusion=...): the batch carries the collated,
        # un-split cloud 'points{i}' of each copy, and the StVD input front end (preprocess.input_front_end) turns it into the
        # streams' points inside the graph, before the voxelisers
        self.fe = vox.get('input_discard') if vox is not None else None
        self.training = False         # (set by the owner before a capture: bin_num 2 and the shuffle when training)
        self.seed = None              # device int64[1]: the front end's draw of the last replay (written inside the graph)
        if self.fe is not None:
            mm = any(st.sfx.startswith('_mm') for st in self.streams)
            if bool(self.fe['later_fusion']) != mm:
                raise ValueError('input_discard: later_fusion=%s, but the model has the input streams %s (two streams: '
                                 'later_fusion=True, VirConv-T / -S; one fused stream: later_fusion=False, VirConv-L)'
                                 % (self.fe['later_fusion'], [st.sfx for st in self.streams]))
            self.raw = {}             # copy suffix -> [cap, 1+C] input buffer of the un-split cloud
            self.raw_prev = {}

    def copy_sfx(self):
        return [''] + [str(i) for i in range(1, self.copies)]

    def _front_end(self, batch_size, static, seed=None, overflow=None, raw=None):
        """The front end of every copy -> ({stream suffix: its points}, published keys)."""
        fe, pts, pub = self.fe, {}, {}
        for i, c in enumerate(self.copy_sfx()):
            r = preprocess.input_front_end(raw[c], batch_size, self.training, bool(fe['later_fusion']), rate=fe.get('rate', 0.8),
                                           seed=seed, point_cloud_range=self.vox['point_cloud_range'], draw=i, static=static,
                                           overflow=overflow)
            pts[c] = r['points']
            pub['stvd_input_kept' + c] = r['stvd_input_kept']
            pub['stvd_input_status' + c] = r['stvd_input_status']
            if fe['later_fusion']:
                pts['_mm' + c] = r['points_mm']
                pub['stvd_input_kept_mm' + c] = r['stvd_input_kept_mm']
        return pts, pub

    def _voxelize(self, st, points, batch_size, static=False):
        v = self.vox
        return ops.voxelize_mean(points, batch_size, v['point_cloud_range'], v['voxel_size'], v['max_points_per_voxel'],
                                 self.vox_arg(st, 'max_voxels'), self.vox_arg(st, 'vfe_model'), static=static)

    def exact_batch(self, batch):
        """`batch` as an exact (host-synchronised) run takes it: with the voxeliser, every stream's points voxelised."""
        bd = dict(batch)
        if self.vox is not None:
            if self.fe is not None:
                pts, pub = self._front_end(int(batch['batch_size']), False, raw={c: batch['points' + c] for c in self.copy_sfx()})
                bd.update(pub)
                bd.update({'points' + s: p for s, p in pts.items()})
            for st in self.streams:
                f, c, _ = self._voxelize(st, bd['points' + st.sfx], int(batch['batch_size']))
                bd.update({'voxel_features' + st.sfx: f, 'voxel_coords' + st.sfx: c})
        return bd

    def allocate(self, batch, dev, margin, grain):
        """(Re)allocate every buffer for `batch`; the input capacities only grow."""
        B = int(batch['batch_size'])
        if self.fe is not None:
            for c in self.copy_sfx():
                pts = batch['points' + c]
                cap = max(self.raw[c].shape[0] if c in self.raw else 0, _round(pts.shape[0], margin, grain))
                row = torch.zeros(pts.shape[1], dtype=torch.float32)
                row[0] = B - 1
                row[1:4] = -1.0e6             # unused tail rows: indicator 0, neither LiDAR nor virtual (the front end drops them)
                self.raw_sentinel = row.to(dev)
                self.raw[c] = self.raw_sentinel.repeat(cap, 1).contiguous()
                self.raw_prev[c] = 0
        for st in self.streams:
            if self.fe is not None:
                st.cap0 = B * int(self.vox_arg(st, 'max_voxels'))
            elif self.vox is not None:
                pts = batch['points' + st.sfx]
                st.cap_pts = max(st.cap_pts, _round(pts.shape[0], margin, grain))
                row = torch.zeros(pts.shape[1], dtype=torch.float32)
                row[0] = B - 1
                row[1:4] = -1.0e6             # unused tail rows: last sample, out of range (the voxeliser drops them)
                st.sentinel = row.to(dev)
                st.pts = st.sentinel.repeat(st.cap_pts, 1).contiguous()
                st.cap0 = B * int(self.vox_arg(st, 'max_voxels'))
            else:
                vf = batch['voxel_features' + st.sfx]
                st.cap0 = max(st.cap0, _round(vf.shape[0], margin, grain))
                st.vf = torch.zeros((st.cap0, vf.shape[1]), dtype=torch.float32, device=dev)
                st.vc = torch.full((st.cap0, 4), -1, dtype=torch.int32, device=dev)
            st.prev_n = 0
        ns = len(self.streams) + self.extra_counts
        self.B = B
        self.n_dev = torch.zeros(ns, dtype=torch.int32, device=dev)
        self.proj = torch.zeros((self.copies, B, 28), dtype=torch.float32, device=dev)
        # pinned staging for the small per-call host values: a ring of slots, each guarded by an event recorded after its
        # upload — the host runs several replays ahead of the GPU, and rewriting ONE pinned buffer before the previous
        # call's asynchronous copy has executed would hand that call the next call's row counts / projection
        self.proj_host = torch.zeros((self.SLOTS, self.copies, B, 28), dtype=torch.float32).pin_memory()
        self.n_host = torch.zeros((self.SLOTS, ns), dtype=torch.int32).pin_memory()
        self._stage_ev, self._stage = [None] * self.SLOTS, 0

    def fits(self, batch):
        """Every stream of `batch` fits the input buffers."""
        if self.fe is not None:
            return all(batch['points' + c].shape[0] <= self.raw[c].shape[0] for c in self.copy_sfx())
        key = 'points' if self.vox is not None else 'voxel_features'
        return all(batch[key + st.sfx].shape[0] <= (st.cap_pts if self.vox is not None else st.cap0) for st in self.streams)

    def load(self, batch, transforms):
        """Copy one batch into the buffers (asynchronous, current stream), with `transforms` (one per copy) for the projection
        blocks; False (nothing copied) when a stream does not fit.  Rows a larger earlier batch left behind are reset to the
        tail values, so that the voxeliser drops them and the published input index set (x_conv1's indices, which are the
        coordinate buffer) keeps its -1 tail."""
        if not self.fits(batch):
            return False
        if self.fe is None:
            key = 'points' if self.vox is not None else 'voxel_features'
            ns = [batch[key + st.sfx].shape[0] for st in self.streams]
        slot = self._stage
        self._stage = (slot + 1) % self.SLOTS
        if self._stage_ev[slot] is not None:
            self._stage_ev[slot].synchronize()         # (8 calls back: has long completed unless the GPU is far behind)
        if self.fe is not None:
            for c in self.copy_sfx():
                n = batch['points' + c].shape[0]
                self.raw[c][:n].copy_(batch['points' + c], non_blocking=True)
                if self.raw_prev[c] > n:
                    self.raw[c][n:self.raw_prev[c]] = self.raw_sentinel
                self.raw_prev[c] = n
            ns = []
        for st, n in zip(self.streams, ns):
            if self.vox is not None:
                st.pts[:n].copy_(batch['points' + st.sfx], non_blocking=True)
                if st.prev_n > n:
                    st.pts[n:st.prev_n] = st.sentinel
            else:
                st.vf[:n].copy_(batch['voxel_features' + st.sfx], non_blocking=True)
                st.vc[:n].copy_(batch['voxel_coords' + st.sfx], non_blocking=True)     # (float32 coordinates -> int32)
                if st.prev_n > n:
                    st.vf[n:st.prev_n] = 0
                    st.vc[n:st.prev_n] = -1
                self.n_host[slot, st.i] = n
            st.prev_n = n
        if self.vox is None:
            self.n_dev.copy_(self.n_host[slot], non_blocking=True)
        for i, trans in enumerate(transforms):
            self.proj_host[slot, i].copy_(torch.from_numpy(ops.projection_params_host(batch['calib'], trans, self.B)))
        self.proj.copy_(self.proj_host[slot], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._stage_ev[slot] = ev
        return True

    def static_batch(self, batch, overflow=None):
        """-> (`batch` with every stream's inputs replaced by the capacity-sized ones, {stream suffix: device int32[1] row
        count}); with the voxeliser, vc_voxelize_mean runs here (inside the graph) once per stream, after the StVD input front
        end (one fresh seed per replay from torch's CUDA generator, kept in `seed`; its overflow word `overflow`) when the
        voxeliser dict asks for it."""
        drop = {k + st.sfx for st in self.streams for k in ('voxel_features', 'voxel_coords', 'points')}
        bd = {k: v for k, v in batch.items() if k not in drop}
        counts = {}
        pts = {st.sfx: getattr(st, 'pts', None) for st in self.streams}
        if self.fe is not None:
            self.seed = torch.randint(preprocess._I64.min, preprocess._I64.max, (1,), dtype=torch.int64, device=self.n_dev.device)
            pts, pub = self._front_end(self.B, True, seed=self.seed, overflow=overflow, raw=self.raw)
            bd.update(pub)
            bd['stvd_input_seed'] = self.seed
        for st in self.streams:
            if self.vox is not None:
                f, c, bd['voxel_num_points' + st.sfx], counts[st.sfx] = self._voxelize(st, pts[st.sfx], self.B, static=True)
            else:
                f, c, counts[st.sfx] = st.vf, st.vc, self.n_dev[st.i:st.i + 1]
            bd.update({'voxel_features' + st.sfx: f, 'voxel_coords' + st.sfx: c})
        return bd, counts


class _Flags:
    """The overflow flags of a captured graph's StaticSpecs (`overflow`, one per plan key) and the library's error flag, read
    back after every replay through a ring of pinned slots, each guarded by an event: the host looks at a replay's flags
    once its event has fired, without waiting for the GPU.  Every replay that overflowed is appended to `events` as {plan
    key: rows that did not fit}."""

    SLOTS = 8

    def __init__(self, keys, dev, events):
        self.keys, self.dev, self.events = list(keys), dev, events
        self.overflow = torch.zeros(len(self.keys), dtype=torch.int32, device=dev)
        self.ovf_host = torch.zeros((self.SLOTS, len(self.keys)), dtype=torch.int32).pin_memory()
        self.err_host = torch.zeros(self.SLOTS, dtype=torch.int32).pin_memory()
        self.pending, self.slot = [], 0      # (event, slot) of the replays whose flags have not been looked at yet

    def flag(self, key):
        """The device int32[1] overflow flag of plan `key` (for its StaticSpec)."""
        j = self.keys.index(key)
        return self.overflow[j:j + 1]

    def wait_if_full(self):
        """With every slot in flight (the host far ahead of the GPU), wait for the oldest replay's flags -> whether it waited."""
        if len(self.pending) < self.SLOTS:
            return False
        self.pending[0][0].synchronize()
        return True

    def push(self):
        """After a replay (current stream): copy its flags into the next slot, zero `overflow`, record the slot's event
        (waiting first when every slot is in flight) -> the event."""
        self.wait_if_full()
        slot = self.slot
        self.slot = (slot + 1) % self.SLOTS
        self.ovf_host[slot].copy_(self.overflow, non_blocking=True)
        self.err_host[slot:slot + 1].copy_(ops.tc_error_flag(self.dev), non_blocking=True)
        self.overflow.zero_()
        ev = torch.cuda.Event()
        ev.record()
        self.pending.append((ev, slot))
        return ev

    def worst(self):
        """The largest overflow, over every flag, of the replays whose flags have arrived (never blocks)."""
        worst = 0
        while self.pending and self.pending[0][0].query():
            slot = self.pending.pop(0)[1]
            if int(self.err_host[slot]) != 0:
                raise _lib.VirConvLibraryError("a tensor-core kernel's pipeline wait timed out inside a replay (error flag "
                                               "set): the results of that replay are invalid")
            vals = [int(v) for v in self.ovf_host[slot]]
            if max(vals):
                self.events.append({k: v for k, v in zip(self.keys, vals) if v})
            worst = max(worst, max(vals))
        return worst


class _Captured:
    """What GraphedStep, PipelinedStep's buffer sets and GraphedForward share: the input side (`inputs`, an _Inputs), the
    StaticSpec capacities of every plan (`caps`, {plan key: {index set: rows}}), the flag ring (`flags`) and the capture
    sequence (_capture).  A subclass sets `inputs` and defines _recapture(batch) and _transforms(batch) (the projection
    transform of each copy)."""

    FE_FLAG = 'stvd_input'    # flag-ring key of the StVD input front end's overflow word

    def __init__(self, dev, voxelizer, margin, grain, warmup):
        self.dev = dev
        self.vox = dict(voxelizer) if voxelizer is not None else None
        self.margin, self.grain, self.warmup = margin, grain, warmup
        self.caps = {}
        self.graphs = []
        self.flags = None
        self.recaptures = 0
        self.launches_per_replay = 0
        self.overflow_events = []         # {plan key: rows that did not fit} of every replay that overflowed

    @property
    def streams(self):
        return self.inputs.streams

    @property
    def ovf_host(self):
        """[8, plan] pinned: the overflow flags of the last replays, one slot each."""
        return self.flags.ovf_host

    def _vox_arg(self, st, key):
        """Voxeliser setting `key` for input stream `st`.  The virtual-point streams ('_mm', '_mm1', ...) read the '_mm' entry
        where the dict has it, and their VFE defaults to the plain mean: the reference's MeanVFE applies its MODEL to the
        LiDAR stream only (mean_vfe.py:51-58).  Every other stream reads the base entry."""
        if st.sfx.startswith('_mm'):
            if key + '_mm' in self.vox:
                return self.vox[key + '_mm']
            if key == 'vfe_model':
                return None
        return self.vox[key]

    def _fe_flag(self):
        return self.flags.flag(self.FE_FLAG) if self.inputs.fe is not None else None

    def _load(self, batch):
        return self.inputs.load(batch, self._transforms(batch))

    def _grow(self, batch):
        self.margin *= 1.25
        self._recapture(batch)

    def _capture(self, batch, exact, warm, bodies, prepare=None):
        """Capture `bodies` (callables of the batch) as one CUDA graph each, in order, for `batch` -> their results; the
        graphs go to `graphs`.  exact(batch) runs the batch exactly and returns {plan key: its executor.last_run}, which
        sizes the plans' capacities (they only grow) and the flag ring; the buffers are sized from the batch, which is
        loaded; warm(batch) runs `warmup` times on a side stream (allocator pools, lazy kernel attributes, arena sizes), as
        torch.cuda.graphs asks for; prepare() runs after it, outside any graph."""
        torch.cuda.synchronize(self.dev)
        self.graphs = []
        self.inputs.training = self.model.training
        runs = exact(batch)
        for key, run in runs.items():
            caps = self.caps.setdefault(key, {})
            for k, v in executor.measured_caps(run, self.margin, self.grain).items():
                caps[k] = max(caps.get(k, 0), v)
        self.inputs.allocate(batch, self.dev, self.margin, self.grain)
        self.flags = _Flags(list(runs) + ([self.FE_FLAG] if self.inputs.fe is not None else []), self.dev, self.overflow_events)
        assert self._load(batch)
        s = torch.cuda.Stream(device=self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s):
            for _ in range(max(self.warmup, 1)):
                warm(batch)
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        if prepare is not None:
            prepare()
        self.flags.overflow.zero_()
        lib = _lib.load()
        l0 = lib.vc_launch_count()
        graphs, outs = [], []
        # A CUDA graph destroyed during a capture invalidates it: torch frees a graph with CUDA calls that the capture mode
        # refuses.  A graph of an earlier step left in an unreachable reference cycle is freed whenever the cyclic collector
        # next runs, so collect such garbage here and keep the collector off until the captures end.
        gc.collect()
        gc_was_on = gc.isenabled()
        gc.disable()
        try:
            for body in bodies:
                graphs.append(torch.cuda.CUDAGraph())
                with torch.cuda.graph(graphs[-1]):
                    outs.append(body(batch))
        finally:
            if gc_was_on:
                gc.enable()
        self.launches_per_replay = int(lib.vc_launch_count() - l0)     # this library's kernels inside one replay
        self.graphs = graphs
        self.recaptures += 1
        torch.cuda.synchronize(self.dev)
        return outs


class GraphedStep(_Captured):
    def __init__(self, model, loss_fn, params=None, margin=1.3, grain=1024, warmup=2, check_overflow=True, voxelizer=None,
                 optimizer=None, max_grad_norm=None):
        """voxelizer: None — batches carry `voxel_features` / `voxel_coords` (what the reference's dataloader + MeanVFE
        deliver); or a dict(point_cloud_range, voxel_size, max_points_per_voxel, max_voxels, vfe_model) — batches carry the
        collated raw `points` [N, 1+C] and the hash-grid voxelisation + VFE (vc_voxelize_mean) run INSIDE the graph.  With a
        two-stream model the batch also carries `points_mm`, voxelised by a second call with the entries `max_voxels_mm`
        (default: `max_voxels`) and `vfe_model_mm` (default: None, the plain mean).  With the entry
        `input_discard=dict(rate=0.8, later_fusion=...)` the batch carries the collated, un-split cloud `points` (indicator 1
        virtual, 2 LiDAR) instead, and the StVD input front end (preprocess.input_front_end: split, input discard, VirConv-L
        re-fusion, range mask, training shuffle) runs inside the graph before the voxelisers, with one fresh seed per replay
        (published as 'stvd_input_seed', the kept rows as 'stvd_input_kept' / 'stvd_input_kept_mm'); later_fusion=True for a
        two-stream model, False for VirConv-L.  Its overflow word is one more flag of the ring (key 'stvd_input').

        optimizer: None — the caller updates the parameters after each call; or an optim.FusedAdamOneCycle — the captured
        body ends with its two update launches (clipping to `max_grad_norm`, None: no clipping), reading the gradients of
        that replay, with every plan's overflow flag and the tensor-core error flag as guard words: a replay that raised one
        skips its own update (optimizer.skipped_steps()) instead of applying gradients of clamped row sets.  Each call
        stages the optimizer's current lr / mom before the replay, so a scheduler sets them as it does for an eager step.
        The exact and warm-up runs of a capture update nothing, and a re-capture keeps the optimizer's state.  Parameters are
        updated in place at fixed addresses: the executor re-casts its bf16 operands from them in every replay, so the next
        replay computes with the new weights with no further action.  A world size above one is refused: the gradient
        all-reduce has to sit between backward and update (use parallel.allreduce_gradients and the eager step()).

        SyncBatchNorm over more than one rank: the graph replays the exchanges' all-reduces, and every call first agrees with
        the other ranks on whether to grow and re-capture (_call_in_step), so that all ranks re-capture together."""
        self.model, self.loss_fn = model, loss_fn
        self.params = list(model.parameters()) if params is None else list(params)
        super().__init__(self.params[0].device, voxelizer, margin, grain, warmup)
        if optimizer is not None and torch.distributed.is_available() and torch.distributed.is_initialized() \
                and torch.distributed.get_world_size() > 1:
            raise ValueError('GraphedStep(optimizer=...) updates inside the graph, before any gradient all-reduce could run: with '
                             'a world size of %d call parallel.allreduce_gradients and the optimizer\'s eager step()'
                             % torch.distributed.get_world_size())
        self.optimizer, self.max_grad_norm = optimizer, max_grad_norm
        self._binding = None          # the optimizer's segment table of the current capture (set by _bind_optimizer)
        self.check_overflow = check_overflow
        self._group = None            # (SyncBatchNorm across ranks, its process group): _rank_group, on the first call
        self.inputs = _Inputs(getattr(model, 'static_streams', ('',)), self.vox, self._vox_arg)

    @property
    def cap0(self):
        """Input row capacity of the first (for VirConvL8x: the only) stream."""
        return self.streams[0].cap0

    def _transforms(self, batch):
        return [batch.get('aug_param')]

    def _clear_grads(self):
        for p in self.params:
            p.grad = None

    def _exact(self, batch):
        """One ordinary (exact-shape, host-synchronised) step -> the row counts of each stream's plan run."""
        self._clear_grads()
        self.loss_fn(self.model(self.inputs.exact_batch(batch))).backward()
        runs = {st.sfx: executor.last_run(self.model, st.sfx) for st in self.streams}
        assert all(r is not None for r in runs.values()), \
            'a captured step needs a backbone running each stream through the plan executor'
        return runs

    def _static_batch(self, batch):
        bd, counts = self.inputs.static_batch(batch, self._fe_flag())
        for st in self.streams:
            bd['virconv_static' + st.sfx] = executor.StaticSpec(counts[st.sfx], self.caps[st.sfx], self.flags.flag(st.sfx),
                                                                alias_params=True)
        bd['virconv_proj'] = self.inputs.proj[0]
        return bd

    def _static_step(self, batch):
        bd = self._static_batch(batch)
        loss = self.loss_fn(self.model(bd))
        # torch.autograd.grad w.r.t. the per-call leaf aliases the executor made of the parameters (executor.run_plan): no
        # long-lived AccumulateGrad node (which remembers the stream it was created on) takes part in a captured backward
        alias = {}
        for st in self.streams:
            alias.update(bd['virconv_static' + st.sfx].param_aliases)
        grads = torch.autograd.grad(loss, [alias.get(id(p), p) for p in self.params], allow_unused=True)
        for p, g in zip(self.params, grads):
            p.grad = g
        if self._binding is not None:
            self._binding.set_grads([p.grad for p in self.optimizer.all_params])
            self._binding.launch(self.max_grad_norm)
        return loss.detach()

    def _warm(self, batch):
        self._clear_grads()
        self._static_step(batch)

    def _bind_optimizer(self):
        # after the warm-up runs (which update nothing: no binding yet), outside the graph: the table's buffers and the
        # guard words of this capture's flags
        self._clear_grads()
        if self.optimizer is not None:
            self._binding = self.optimizer.bind([self.flags.overflow, ops.tc_error_flag(self.dev)])

    def _recapture(self, batch):
        self._binding = None
        self.loss, = self._capture(batch, self._exact, self._warm, [self._static_step], self._bind_optimizer)

    def _rank_group(self):
        """(True, process group) when the model's SyncBatchNorm layers exchange over more than one rank, else (False, None)."""
        if self._group is None:
            sync = [m for m in self.model.modules() if isinstance(m, torch.nn.SyncBatchNorm)]
            self._group = (True, sync[0].process_group) if sync and sync_bn.world_size(sync) > 1 else (False, None)
        return self._group

    def _call_in_step(self, batch, group):
        """__call__ under SyncBatchNorm across ranks.  A re-capture runs eager steps whose exchanges are real collectives, so
        the ranks must grow and re-capture together: the decision is one all-reduce (MAX) of [largest overflow so far, this
        batch does not fit], taken after the previous replay has finished (its flags are then in on every rank).  This waits
        for the previous replay on every call: the host does not run ahead of the GPU in this mode."""
        torch.cuda.current_stream(self.dev).synchronize()
        worst = self.flags.worst() if self.check_overflow else 0
        vote = torch.tensor([worst, 0 if self.inputs.fits(batch) else 1], dtype=torch.int32, device=self.dev)
        torch.distributed.all_reduce(vote, op=torch.distributed.ReduceOp.MAX, group=group)
        if max(vote.tolist()):
            self._grow(batch)
        assert self._load(batch)
        self.graphs[0].replay()
        if self.check_overflow:
            self.flags.push()
        return self.loss

    def __call__(self, batch):
        """-> the step's loss (a device tensor owned by the graph: read or copy it before the next call)."""
        if not self.graphs:
            self._recapture(batch)
        sync, group = self._rank_group()
        if sync:
            return self._call_in_step(batch, group)
        if self.optimizer is not None:
            self.optimizer.stage_hyper()
            if self.check_overflow:
                # look at the oldest replay's flags BEFORE this replay, not after it: a batch whose update ran inside the graph
                # must not run a second time
                self.flags.wait_if_full()
        if self.check_overflow and self.flags.worst():
            # an EARLIER batch did not fit: its gradients were computed on clamped row sets.  Grow and re-capture; the
            # caller sees the event through `recaptures` (a training loop may want to discard those optimizer steps).
            self._grow(batch)
        if not self._load(batch):
            self._grow(batch)               # more input rows than the input buffers hold
            assert self._load(batch)
        self.graphs[0].replay()
        if self.check_overflow:
            if self.flags.wait_if_full() and self.flags.worst():
                self._grow(batch)
                return self(batch)
            self.flags.push()
        return self.loss


class _PipeInstance(GraphedStep):
    """One of the two buffer sets of a PipelinedStep: the step captured as TWO graphs over one caller-owned arena — the index
    graph (voxeliser, rulebooks, projections: everything that depends on coordinates only) and the feature graph (weight images,
    conv + BN + ReLU, loss, backward)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.feat_done = None
        self.grads = None

    def _index_part(self, batch):
        bd = self._static_batch(batch)              # (in-graph voxeliser, if any)
        spec = bd['virconv_static']
        spec.phase, spec.arena = 1, self.arena
        self.model.index_phase(bd)
        self._bd = bd                               # (the feature graph continues from it)

    def _feature_part(self, batch):
        spec = self._bd['virconv_static']
        spec.phase = 2
        loss = self.loss_fn(self.model(self._bd))
        alias = spec.param_aliases
        grads = torch.autograd.grad(loss, [alias.get(id(p), p) for p in self.params], allow_unused=True)
        self.grads = list(grads)
        return loss.detach()

    def _prepare(self):
        # the arena both graphs share, sized from what the (unphased) warm-up steps used
        plan = self.model._plan()
        self.arena = executor.empty_scratch(executor._arena_bytes(plan, self.cap0, self.dev, True), torch.uint8, self.dev)
        self._clear_grads()

    def _recapture(self, batch):
        _, self.loss = self._capture(batch, self._exact, self._warm, [self._index_part, self._feature_part], self._prepare)
        self.feat_done = None


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
        if kwargs.get('optimizer') is not None:
            raise ValueError('PipelinedStep overlaps the index work of step t+1 with the feature work of step t and has no '
                             'in-graph update: pass optimizer= to GraphedStep, or call the optimizer\'s step() after each call')
        if (kwargs.get('voxelizer') or {}).get('input_discard') is not None:
            raise ValueError('PipelinedStep does not run the StVD input front end (voxelizer input_discard): use GraphedStep')
        if sync_bn.world_size(list(model.modules())) > 1:
            raise ValueError('PipelinedStep runs the feature phase of step t beside the index phase of step t+1 and has no '
                             'SyncBatchNorm exchange across ranks: use GraphedStep')
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
        if not inst.graphs:
            inst._recapture(batch)
        if inst.check_overflow and inst.flags.worst():
            inst._grow(batch)
        with torch.cuda.stream(self.s_idx):
            if inst.feat_done is not None:
                self.s_idx.wait_event(inst.feat_done)          # the buffer set's previous step (two steps back) is through
            else:
                self.s_idx.wait_stream(main)
            ok = inst._load(batch)
            if ok:
                inst.graphs[0].replay()
                ev = torch.cuda.Event()
                ev.record(self.s_idx)
        if not ok:                                             # more input rows than the buffers hold: grow, re-capture, run again
            inst._grow(batch)
            self.t -= 1
            return self(batch)
        main.wait_event(ev)
        inst.graphs[1].replay()
        for p, g in zip(self.params, inst.grads):
            p.grad = g
        if inst.check_overflow:
            inst.flags.push()
        inst.feat_done = torch.cuda.Event()
        inst.feat_done.record(main)
        return inst.loss


class GraphedForward(_Captured):
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
    `margin`; a re-capture with the same number of copies only grows them), and its own overflow flag.
    check_overflow='sync' (default): each call reads this replay's overflow and error flags before returning; a batch that
    did not fit is re-run after a re-capture with larger capacities, so a returned result never comes from clamped row sets.
    'async': the flags are read one call late, as GraphedStep does (the result of an overflowing batch is then returned, and
    `recaptures` grows on the next call).

    voxelizer: as GraphedStep's — the batch then carries 'points{i}' (and 'points_mm{i}' for VirConv8x with MM) instead of the
    voxel keys, and vc_voxelize_mean runs inside the graph once per stream and copy; the virtual-point stream's settings are
    the '_mm' entries ('max_voxels_mm', 'vfe_model_mm', default the plain mean).  With the voxeliser's `input_discard` entry
    (GraphedStep) the batch carries the un-split collated cloud 'points{i}' of each copy; each copy goes through the StVD
    input front end independently (its own draw under the replay's seed, bin_num 10, no shuffle: the test-time settings)."""

    def __init__(self, model, margin=1.3, voxelizer=None, bev=False, check_overflow='sync', grain=1024, warmup=2):
        from .backbone import VirConv8x, VirConvL8x
        if not isinstance(model, (VirConv8x, VirConvL8x)):
            raise ValueError('GraphedForward captures a VirConvL8x or VirConv8x backbone, got %s' % type(model).__name__)
        if model.training:
            raise ValueError('GraphedForward captures the test-time forward: call model.eval() first (a captured training step '
                             'is graph.GraphedStep)')
        if check_overflow not in ('sync', 'async'):
            raise ValueError("check_overflow: 'sync' or 'async', got %r" % (check_overflow,))
        super().__init__(next(model.parameters()).device, voxelizer, margin, grain, warmup)
        self.model = model
        self.x_batched = isinstance(model, VirConv8x)
        self.mm = self.x_batched and model.mm
        self.bev, self.check_overflow = bool(bev), check_overflow
        self.R = None
        self.inputs = None

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
        if self.vox is not None and self.vox.get('input_discard') is not None:
            missing = ['points' + s for s in self._sfx(R) if batch.get('points' + s) is None]      # the un-split clouds
        else:
            missing = [k + s for s in self.input_streams(R) for k in keys if batch.get(k + s) is None]
        if missing:
            raise ValueError('GraphedForward: the batch has no %s' % ', '.join(missing))
        return R

    def _transforms(self, batch):
        tp = batch.get('transform_param')
        return [tp[:, i, :] if tp is not None else batch.get('aug_param') for i in range(self.R)]

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
        """One exact eager eval forward (host-synchronised) -> the row counts of every plan run."""
        executor._LAST_RUNS.pop(self.model, None)
        bd = self.inputs.exact_batch(batch)
        with torch.no_grad():
            self.model(bd)
        runs = {k: executor.last_run(self.model, k) for k in self.plan_streams(self.R)}
        if any(r is None for r in runs.values()):
            from .backbone import _module_path_reason
            raise ValueError('GraphedForward: the eval forward does not run through the plan executor (%s)'
                             % _module_path_reason(bd['voxel_features' + self.streams[0].sfx]))
        return runs

    @torch.no_grad()
    def _static_forward(self, batch):
        from .backbone import EvalStaticSpec
        bd, counts = self.inputs.static_batch(batch, self._fe_flag())
        flag = self.flags.flag
        if self.x_batched:
            sfx = self._sfx(self.R)
            lidar = executor.StaticSpec(self.inputs.n_dev[-1:], self.caps[''], flag(''))
            mm = [executor.StaticSpec(counts['_mm' + s], self.caps['_mm' + s], flag('_mm' + s)) for s in sfx] if self.mm else []
            bd['virconv_eval_static'] = EvalStaticSpec(lidar, [counts[s] for s in sfx], mm, self.inputs.proj)
        else:
            bd['virconv_static'] = executor.StaticSpec(counts[''], self.caps[''], flag(''))
            bd['virconv_proj'] = self.inputs.proj[0]
        before = set(bd)
        out = self.model(bd)
        if self.bev:
            self._bev(out)
        self._published = [k for k in out if k not in before or k.startswith('stvd_input')]
        return out

    def _recapture(self, batch):
        self.out, = self._capture(batch, self._exact, self._static_forward, [self._static_forward])

    # -- replay ----------------------------------------------------------------------------------------------------
    def __call__(self, batch):
        """-> the batch dict plus the published tensors of this forward (owned by the graph: valid until the next call)."""
        R = self.copies(batch)
        if R != self.R:
            # other copies, other streams and plans: buffers and capacities start afresh
            self.R, self.caps = R, {}
            # (n_dev[-1]: the packed LiDAR rows, written in the graph)
            self.inputs = _Inputs(self.input_streams(R), self.vox, self._vox_arg, copies=R, extra_counts=1)
            self.graphs = []
        if not self.graphs or int(batch['batch_size']) != self.inputs.B:
            self._recapture(batch)
        if self.check_overflow == 'async' and self.flags.worst():
            self._grow(batch)              # an EARLIER batch did not fit: its result came from clamped row sets
        while True:
            if not self._load(batch):
                self._grow(batch)          # more input rows than the buffers hold
                continue
            self.graphs[0].replay()
            if self.check_overflow == 'sync':
                self.flags.push().synchronize()
                if self.flags.worst():
                    self._grow(batch)      # this batch did not fit: re-capture and run it again
                    continue
            else:
                self.flags.push()
            break
        res = dict(batch)
        res.update({k: self.out[k] for k in self._published})
        return res
