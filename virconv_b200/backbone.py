"""VirConv 3-D backbones on the virconv_b200 operators — drop-in for the classes the detector registry
instantiates (`pcdet/models/backbones_3d/__init__.py:3-8`, `detector3d_template.py:65-78`):
same constructor `(model_cfg, input_channels, grid_size, **kwargs)`, same `.forward(batch_dict)` keys,
same `.num_point_features`, same sub-module names (=> same state_dict keys, SURVEY §5).

Restated from `pcdet/models/backbones_3d/spconv_backbone.py`: NRConvBlock :150-229, VirConvL8x :538-699,
layer_voxel_discard :134-147.  Differences that do not change results:
  * conv + BatchNorm1d + ReLU run as one fused op; the d3/d2 conv pairs of a block share one rulebook
    (identical indices) although the reference builds it twice under distinct indice_keys;
  * `index2uv` is one kernel over the whole batch (the reference loops over samples with boolean-mask
    indexing, :61-78); its per-sample matrices are built once per forward;
  * StVD layer discard: `discard_mode='spconv2_compat'` reproduces the reference under spconv 2.x, where
    `layer_voxel_discard` returns None after rebinding a local and the caller's tensor is unchanged
    (SURVEY §5 note) — i.e. no discard; `discard_mode='paper'` really drops rows, order-preserving.  Where the kept rows
    are drawn: `discard_rng='numpy'` (default) from the global numpy stream on the host, as the reference under
    `set_random_seed`, on the per-operator module path; `discard_rng='device'` on the GPU inside the plan executor
    (csrc/stvd_layer.cu: a uniformly random k-subset of the same size, from one int64 seed per forward drawn with
    torch's CUDA generator, or `batch_dict['stvd_seed']`), which a CUDA graph can capture.  Either way the applied lists
    can be fed back through `batch_dict['stvd_keep_rows']`; the device draw records them in `batch_dict['stvd_kept_rows']`.
"""
from __future__ import annotations

import warnings
from functools import partial

import numpy as np

import torch
import torch.nn as nn

from . import executor, ops, sync_bn
from . import spconv_compat as spconv


def _cfg_get(cfg, key, default=None):
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default) if not hasattr(cfg, 'get') else cfg.get(key, default)


norm_fn = partial(nn.BatchNorm1d, eps=1e-3, momentum=0.01)


def sparse_block(cin, cout, kernel_size, norm_fn, ndim=3, conv_type='subm', stride=1, padding=0, indice_key=None):
    """conv(bias=False) -> norm -> ReLU, as post_act_block / post_act_block2d (:86-131)."""
    if conv_type == 'subm':
        cls = spconv.SubMConv3d if ndim == 3 else spconv.SubMConv2d
        conv = cls(cin, cout, kernel_size, bias=False, indice_key=indice_key)
    elif conv_type == 'spconv':
        cls = spconv.SparseConv3d if ndim == 3 else spconv.SparseConv2d
        conv = cls(cin, cout, kernel_size, stride=stride, padding=padding, bias=False, indice_key=indice_key)
    else:
        raise NotImplementedError(conv_type)
    return spconv.SparseSequential(conv, norm_fn(cout), nn.ReLU())


class NRConvBlock(nn.Module):
    """Noise-resistant conv block: [strided down conv] -> 2x SubMConv3d -> project voxels to pixels ->
    2x SubMConv2d in image space -> concat (spconv_backbone.py:150-229)."""

    def __init__(self, input_c=16, output_c=16, stride=1, padding=1, indice_key='vir1', conv_depth=False):
        super().__init__()
        self.stride = stride
        self.conv_depth = conv_depth
        if stride > 1:
            self.down_layer = sparse_block(input_c, output_c, 3, norm_fn, 3, 'spconv', stride, padding,
                                           'sp' + indice_key)
        c1 = output_c if stride > 1 else input_c
        if conv_depth:
            c1 += 4
        half = output_c // 2
        self.d3_conv1 = sparse_block(c1, half, 3, norm_fn, 3, 'subm', padding=1, indice_key='subm1' + indice_key)
        self.d2_conv1 = sparse_block(half, half, 3, norm_fn, 2, 'subm', padding=1, indice_key='subm3' + indice_key)
        self.d3_conv2 = sparse_block(half, half, 3, norm_fn, 3, 'subm', padding=1, indice_key='subm2' + indice_key)
        self.d2_conv2 = sparse_block(half, half, 3, norm_fn, 2, 'subm', padding=1, indice_key='subm4' + indice_key)

    def forward(self, sp_tensor, batch_size, proj_params, stride):
        if self.stride > 1:
            sp_tensor = self.down_layer(sp_tensor)
        idx = spconv._as_i32(sp_tensor.indices)
        rb2d = None
        if ops.OVERLAP and idx.shape[0] > 0:
            # projection + the image-space rulebook only need the indices: build them on the side stream while the two
            # 3-D convs run on the main one
            sd = ops.side(idx.device)
            main = torch.cuda.current_stream()
            sd.stream.wait_stream(main)
            with torch.cuda.stream(sd.stream):
                uv = ops.index2uv(idx, batch_size, proj_params, stride)
                conv2d = self.d2_conv1[0]
                rb2d = ops.build_subm_rulebook(uv, batch_size, [1600, 600], conv2d.kernel_size, conv2d.dilation)
            ops._keep_alive_on(sd.stream, idx, proj_params)
            ops._keep_alive_on(main, uv, rb2d.nbr, rb2d.pair_num)
        d3 = self.d3_conv2(self.d3_conv1(sp_tensor))
        if rb2d is None:
            uv = ops.index2uv(spconv._as_i32(d3.indices), batch_size, proj_params, stride)
        else:
            torch.cuda.current_stream().wait_stream(sd.stream)
        img = spconv.SparseConvTensor(d3.features, uv, [1600, 600], batch_size)
        if rb2d is not None:
            rb2d._keepalive = uv
            img.indice_dict[self.d2_conv1[0].indice_key] = rb2d       # both image convs see identical indices
            img.indice_dict[self.d2_conv2[0].indice_key] = rb2d
        img.features_bf16 = d3.features_bf16
        d2 = self.d2_conv2(self.d2_conv1(img))
        cat = ops.Cat2Fn.apply(d3.features, d2.features, d3.features_bf16 is not None)
        if isinstance(cat, tuple):
            out = d3.replace_feature(cat[0])
            out.features_bf16 = cat[1]
            return out
        return d3.replace_feature(cat)


def plan_nrconv(plan, block, f, iset, proj_stride):
    """Record one NRConvBlock (NRConvBlock.forward above; spconv_backbone.py:207-229) into an executor plan.  Index ops
    first (they go to the side stream), then the feature ops.  -> (feature slot of the concat, index set of the block)."""
    if block.stride > 1:
        conv = block.down_layer[0]
        iset, rb = plan.conv_rb(iset, 3, conv.kernel_size, conv.stride, conv.padding, conv.dilation, keys=[conv.indice_key])
        f = plan.cbr(f, rb, conv, block.down_layer[1], seq=block.down_layer)
    c3, c2 = block.d3_conv1[0], block.d2_conv1[0]
    assert (block.d3_conv2[0].kernel_size, block.d3_conv2[0].dilation) == (c3.kernel_size, c3.dilation)
    assert (block.d2_conv2[0].kernel_size, block.d2_conv2[0].dilation) == (c2.kernel_size, c2.dilation)
    rb3 = plan.subm_rb(iset, 3, c3.kernel_size, c3.dilation, unique=True, keys=[c3.indice_key, block.d3_conv2[0].indice_key],
                       stream=2)        # stream 1 keeps the strided convs' count -> indices -> tables chain to itself
    uv = plan.index2uv(iset, proj_stride, stream=2)
    rb2 = plan.subm_rb(uv, 2, c2.kernel_size, c2.dilation, unique=False,      # projected pixels collide
                       keys=[c2.indice_key, block.d2_conv2[0].indice_key], stream=2)
    d3 = plan.cbr(plan.cbr(f, rb3, c3, block.d3_conv1[1], seq=block.d3_conv1), rb3, block.d3_conv2[0], block.d3_conv2[1],
                  seq=block.d3_conv2)
    d2 = plan.cbr(plan.cbr(d3, rb2, c2, block.d2_conv1[1], seq=block.d2_conv1), rb2, block.d2_conv2[0], block.d2_conv2[1],
                  seq=block.d2_conv2)
    return plan.cat(d3, d2), iset


def _published_tensors(run, res, names, coords0, shape0, batch_size):
    """The named results of a plan run; tensors over index sets of one group (executor.Plan.iset_group) share one lazy
    indice_dict."""
    plan, dicts, out = run.plan, {}, []
    sets = {name: iset for name, _, iset in plan.published}
    for name in names:
        g = plan.iset_group[sets[name]]
        if g not in dicts:
            dicts[g] = executor.LazyIndiceDict(run, coords0, shape0, g)
        out.append(_published_tensor(res, name, batch_size, dicts[g]))
    return tuple(out)


def _published_tensor(res, name, batch_size, indice_dict):
    f, idx, shape, fb, cnt = res[name]
    t = spconv.SparseConvTensor(f, idx, shape, batch_size, indice_dict=indice_dict)
    t.features_bf16 = fb
    t.num_rows = cnt          # static mode: device int32[1] row count (features / indices are capacity sized, zero / -1 tail)
    return t


def stvd_keep_rows(n, rate, rng=np.random):
    """Rows kept by StVD layer discard: the reference draws `np.random.permutation(n)[:int(n*(1-rate))]`
    (:143-144); kept order-preserving (sorted) so published tensors stay batch-contiguous."""
    keep = rng.permutation(n)[:int(n * (1 - rate))]
    return np.sort(keep)


_I64 = torch.iinfo(torch.int64)


def stvd_seed(batch_dict, device):
    """The draw behind one forward's device-side layer discards: batch_dict['stvd_seed'] (int64 device tensor) when given,
    else one int64 from torch's CUDA generator on the current stream — fresh on every replay of a captured graph, repeated
    under torch.manual_seed."""
    seed = batch_dict.get('stvd_seed')
    if seed is None:
        return torch.randint(_I64.min, _I64.max, (1,), dtype=torch.int64, device=device)
    assert torch.is_tensor(seed) and seed.dtype == torch.int64 and seed.device == device and seed.numel() == 1, \
        "batch_dict['stvd_seed'] must be one int64 on the model's device"
    return seed.reshape(1)


def discard_rows(t, keep_rows):
    if torch.is_tensor(keep_rows):      # a list the device draw recorded (static mode: capacity-sized, count in .num_rows)
        n = getattr(keep_rows, 'num_rows', None)
        rows = (keep_rows if n is None else keep_rows[:int(n)]).to(device=t.features.device, dtype=torch.int32).contiguous()
    else:
        rows = torch.as_tensor(np.ascontiguousarray(keep_rows), dtype=torch.int32).to(t.features.device)
    feats = ops.GatherRowsFn.apply(t.features, rows)
    idx = ops.gather_rows(spconv._as_i32(t.indices), rows)
    return spconv.SparseConvTensor(feats, idx, t.spatial_shape, t.batch_size)


def _copy_transform(batch_dict, i):
    """The augmentation of transformed copy i: transform_param[:, i] (X_TRANS copies), else aug_param."""
    if 'transform_param' in batch_dict:
        return batch_dict['transform_param'][:, i, :]
    return batch_dict.get('aug_param')


def _publish(batch_dict, sfx, xs, out=None, stream=''):
    """The keys the detector reads for copy `sfx`: x_conv1..4 (`xs`; None where the eval forward of VirConv8x publishes
    none) and the encoded tensor `out`.  stream='_mm': VirConv8x's virtual-point stream, which has no encoded tensor and puts
    '_mm' before the copy suffix — but not in its strides key, as the reference writes it (spconv_backbone.py:527)."""
    if out is not None:
        batch_dict['encoded_spconv_tensor' + sfx] = out
    batch_dict.update({
        'encoded_spconv_tensor_stride' + stream + sfx: 8,
        'multi_scale_3d_features' + stream + sfx: dict(zip(('x_conv1', 'x_conv2', 'x_conv3', 'x_conv4'), xs)),
        'multi_scale_3d_strides' + sfx: {'x_conv1': 1, 'x_conv2': 2, 'x_conv3': 4, 'x_conv4': 8},
    })


class _VirConvBackbone(nn.Module):
    """What VirConvL8x and VirConv8x share: the config, conv_out, and the virtual-point stream — vir_conv1..4 with the StVD
    layer discards — run through a cached executor plan or on the per-operator module path."""

    # VirConv8x also discards the stream's input voxels (:489-490): discard site 0, the blocks' sites follow it
    _input_discard = False

    def __init__(self, model_cfg, grid_size, discard_mode, discard_rng):
        super().__init__()
        self.model_cfg = model_cfg
        self.return_num_features_as_dict = _cfg_get(model_cfg, 'RETURN_NUM_FEATURES_AS_DICT', False)
        self.out_features = _cfg_get(model_cfg, 'OUT_FEATURES', 64)
        self.layer_discard_rate = _cfg_get(model_cfg, 'LAYER_DISCARD_RATE', 0.0)
        self.num_filters = list(_cfg_get(model_cfg, 'NUM_FILTERS', [16, 32, 64, 64]))
        assert discard_mode in ('spconv2_compat', 'paper')
        assert discard_rng in ('numpy', 'device')
        self.discard_mode, self.discard_rng = discard_mode, discard_rng
        gs = [int(g) for g in grid_size]
        self.sparse_shape = [gs[2] + 1, gs[1], gs[0]]            # grid_size[::-1] + [1, 0, 0]   (:552)
        self.num_point_features = self.out_features
        if self.return_num_features_as_dict:
            self.num_point_features = {'x_conv%d' % (i + 1): self.num_filters[i] for i in range(4)}

    def _add_nrconv_blocks(self, input_channels):
        f = self.num_filters
        self.vir_conv1 = NRConvBlock(input_channels, f[0], stride=1, indice_key='vir1')
        self.vir_conv2 = NRConvBlock(f[0], f[1], stride=2, indice_key='vir2')
        self.vir_conv3 = NRConvBlock(f[1], f[2], stride=2, indice_key='vir3')
        self.vir_conv4 = NRConvBlock(f[2], f[3], stride=2, padding=(0, 1, 1), indice_key='vir4')

    def _add_conv_out(self):
        last_pad = _cfg_get(self.model_cfg, 'last_pad', 0)
        self.conv_out = spconv.SparseSequential(
            spconv.SparseConv3d(self.num_filters[3], self.out_features, (3, 1, 1), stride=(2, 1, 1), padding=last_pad,
                                bias=False, indice_key='spconv_down2'),
            norm_fn(self.out_features), nn.ReLU())

    # -- StVD layer discard ----------------------------------------------------------------------------------
    def _discarding(self):
        return self.training and self.discard_mode == 'paper' and self.layer_discard_rate != 0

    def _device_discard(self):
        return self._discarding() and self.discard_rng == 'device'

    def _host_discard(self, batch_dict):
        """Kept rows drawn on the host or given in batch_dict['stvd_keep_rows']: applied on the module path (a device draw
        runs in the plan)."""
        return self._discarding() and (self.discard_rng != 'device' or batch_dict.get('stvd_keep_rows') is not None)

    def _maybe_discard(self, t, batch_dict, site):
        if not self._discarding():
            return t
        given = batch_dict.get('stvd_keep_rows')
        keep = given[site] if given is not None else stvd_keep_rows(t.features.shape[0], self.layer_discard_rate)
        return discard_rows(t, keep)

    # -- SyncBatchNorm (sync_bn): `bn_reducer` replaces the all-reduce of the exchanged BN sums ---------------------
    bn_reducer = None

    def _no_module_path_under_sync(self, plan, reason):
        """SyncBatchNorm layers exchanging their sums: every rank must issue the same collectives in the same order.  A reason
        that is the same on every rank (VIRCONV_EXECUTOR=0, host-drawn StVD, the module types) sends every rank to the module
        path, where torch's SyncBatchNorm exchanges in step; a reason that depends on the rank's own batch or call raises
        instead (the other ranks would wait for its plan's exchanges)."""
        if reason in _RANK_DEPENDENT and sync_bn.active(self, [bn for _, bn in plan.layers]):
            raise RuntimeError('VirConv backbone: SyncBatchNorm across ranks runs through the plan executor on every rank, and '
                               'this forward cannot (%s)' % reason)

    # -- native plans (csrc/executor.cu): the whole forward / backward of a stream in one C-ABI call each ------
    def _cached_plan(self, attr, build):
        """The plan cached under `attr`, rebuilt by build() when there is none or it is stale (a sub-module was replaced after
        it was built, e.g. by SyncBatchNorm conversion).  Copies and pickles of the model drop it (executor.Plan)."""
        plan = getattr(self, attr, None)
        if plan is None or not plan.is_current():
            plan = build()
            setattr(self, attr, plan)
        return plan

    def _nrconv_plan(self, stvd):
        """The virtual-point stream as a plan -> (plan, feature slot, index set) of its last block.  stvd: with the
        device-drawn layer discards, numbered in stream order — the input voxels (site 0) where the class discards them, then
        after vir_conv1..3."""
        plan = executor.Plan(self.vir_conv1.d3_conv1[0].in_channels)
        f, iset = 0, 0
        first = int(self._input_discard)
        if stvd and self._input_discard:
            f, iset = plan.discard(f, iset, 0, self.layer_discard_rate)
        for i, (blk, s) in enumerate(zip((self.vir_conv1, self.vir_conv2, self.vir_conv3, self.vir_conv4), (1, 2, 4, 8))):
            f, iset = plan_nrconv(plan, blk, f, iset, s)
            if stvd and i < 3:
                f, iset = plan.discard(f, iset, first + i, self.layer_discard_rate)
            plan.publish('x_conv%d' % (i + 1), f, iset)
        return plan, f, iset

    def _plan_conv_out(self, plan, f, iset):
        """Append conv_out to `plan`, its output published as 'out'."""
        co = self.conv_out[0]
        iset, rb = plan.conv_rb(iset, 3, co.kernel_size, co.stride, co.padding, co.dilation, keys=[co.indice_key])
        plan.publish('out', plan.cbr(f, rb, co, self.conv_out[1], seq=self.conv_out), iset)
        return plan

    def _run(self, plan, feats, coords, shape, batch_size, proj, stream, seed=None, static=None, inputs_ready=False):
        """-> (run record, published tensors).  stream: the executor.note_last_run key of the input stream; static: its
        StaticSpec (capacity-sized feats / coords)."""
        ci = spconv._as_i32(coords)
        run, res = executor.run_plan(plan, feats, ci, shape, batch_size, proj, plan.layers[0][1].training,
                                     plan.layers[0][0].precision, inputs_ready=inputs_ready, static=static, seed=seed,
                                     reducer=sync_bn.reducer_for(self, [bn for _, bn in plan.layers]), tag=stream)
        # (graph.GraphedStep sizes each stream's capacities from an exact run.)  The default stream '' is left to
        # note_last_run's default, so that wrappers of it taking (model, run) keep working for one-stream models
        if stream:
            executor.note_last_run(self, run, stream)
        else:
            executor.note_last_run(self, run)
        return run, _published_tensors(run, res, [name for name, _, _ in plan.published], ci, shape, batch_size)

    def _plan_inputs(self, batch_dict, feats, coords, static, stvd, side):
        """-> (int32 coordinates, StVD seed or None, inputs_ready) of a plan run of the virtual-point stream."""
        return spconv._as_i32(coords), (stvd_seed(batch_dict, feats.device) if stvd else None), False

    def _nrconv_stream(self, batch_dict, plan, feats, coords, trans, sfx, stream, proj=None, static=None, out=None,
                       refusal=None):
        """The virtual-point stream of one copy (batch-key suffix `sfx`, note_last_run key `stream`) -> its published tensors:
        x_conv1..4, then `out`'s (VirConvL8x's conv_out, which `plan` ends with).  Runs `plan` when _module_path_reason
        allows it, else the module path with the same discard sites — or raises ValueError(refusal % reason) when given.
        proj: the [B,28] projection block on the device, else made from batch_dict['calib'] and `trans`; static: the
        StaticSpec of a static-mode run.  A device-drawn discard records its kept rows in 'stvd_kept_rows' + sfx."""
        batch_size = batch_dict['batch_size']
        reason = _module_path_reason(feats, plan, self._host_discard(batch_dict))
        if reason is None:
            side = ops.side(feats.device).stream if executor.TWO_STREAMS else None
            ci, seed, ready = self._plan_inputs(batch_dict, feats, coords, static, bool(plan.discards), side)
            if proj is None:
                assert static is None, "static mode needs batch_dict['virconv_proj'] (ops.projection_params on the device)"
                proj = ops.projection_params(batch_dict.get('calib'), trans, batch_size, feats.device, side)
            run, xs = self._run(plan, feats, ci, self.sparse_shape, batch_size, proj, stream, seed, static, ready)
            if seed is not None:
                batch_dict['stvd_kept_rows' + sfx] = run.kept_rows()
            return xs
        if refusal is not None:
            raise ValueError(refusal % reason)
        self._no_module_path_under_sync(plan, reason)
        _module_path_under_determinism(reason)
        proj = ops.projection_params(batch_dict.get('calib'), trans, batch_size, feats.device)
        x = spconv.SparseConvTensor(feats, coords.int(), self.sparse_shape, batch_size)
        first = int(self._input_discard)
        if self._input_discard:
            x = self._maybe_discard(x, batch_dict, 0)
        xs = []
        for i, (blk, s) in enumerate(zip((self.vir_conv1, self.vir_conv2, self.vir_conv3, self.vir_conv4), (1, 2, 4, 8))):
            x = blk(x, batch_size, proj, s)
            if i < 3:
                x = self._maybe_discard(x, batch_dict, first + i)
            xs.append(x)
        if out is not None:
            xs.append(out(x))
        return tuple(xs)


class VirConvL8x(_VirConvBackbone):
    """VirConv-L backbone (fused LiDAR + virtual stream), spconv_backbone.py:538-699."""

    def __init__(self, model_cfg, input_channels, grid_size, discard_mode='spconv2_compat', precision='fp32',
                 discard_rng='numpy', **kwargs):
        super().__init__(model_cfg, grid_size, discard_mode, discard_rng)
        self._add_nrconv_blocks(input_channels)
        self._add_conv_out()
        spconv.set_precision(self, precision)

    def _plan(self):
        """The plan of the current mode: the virtual-point stream and conv_out, with the three layer discards (sites 0-2,
        after vir_conv1..3) in a device-drawn paper-mode training forward, without them otherwise; both are cached."""
        stvd = self._device_discard()
        return self._cached_plan('_plan_stvd_cache' if stvd else '_plan_cache',
                                 lambda: self._plan_conv_out(*self._nrconv_plan(stvd)))

    def _use_plan(self, feats, batch_dict=None):
        return _module_path_reason(feats, self._plan(), self._host_discard(batch_dict or {})) is None

    def index_phase(self, batch_dict):
        """Phased static execution (graph.PipelinedStep), phase 1: everything of the forward that depends on the voxel
        COORDINATES only — int32 coordinates, rulebooks of every stage, voxel -> pixel projections — enqueued into
        batch_dict['virconv_static'].arena.  forward() with the same batch_dict and `static.phase = 2` then runs the
        feature operators over it."""
        feats, coords = batch_dict['voxel_features'], batch_dict['voxel_coords']
        static = batch_dict['virconv_static']
        assert static.phase == 1 and self._use_plan(feats, batch_dict)
        plan = self._plan()
        ci = spconv._as_i32(coords)
        # (the layer discards select their rows in this phase; the feature phase gathers with the same seed)
        seed = stvd_seed(batch_dict, feats.device) if plan.discards else None
        executor.run_index(plan, feats, ci, self.sparse_shape, batch_dict['batch_size'], batch_dict['virconv_proj'],
                           plan.layers[0][1].training, plan.layers[0][0].precision, static, seed)
        batch_dict['virconv_ci'] = ci
        batch_dict['virconv_stvd_seed'] = seed
        return batch_dict

    def _plan_inputs(self, batch_dict, feats, coords, static, stvd, side):
        if static is not None and static.phase == 2:
            return batch_dict['virconv_ci'], batch_dict['virconv_stvd_seed'], False     # (index_phase of this very batch)
        seed = stvd_seed(batch_dict, feats.device) if stvd else None
        # 'virconv_inputs_ready': the caller's promise that voxel_coords is resident and complete (a prefetched batch) -> the
        # index pipeline of this step (starting with the .int() of the coordinates, :641) runs on the side stream without
        # waiting for main, i.e. it may overlap the previous step's backward
        ready = side is not None and static is None and seed is None and bool(batch_dict.get('virconv_inputs_ready', False))
        if ready and (coords.dtype != torch.int32 or not coords.is_contiguous()):
            executor.reserve_blocks('coords_i32', 4 * coords.numel(), feats.device, side)
            with torch.cuda.stream(side):
                ci = spconv._as_i32(coords)
            ci.record_stream(torch.cuda.current_stream(feats.device))   # published as x_conv1's indices
            return ci, seed, ready
        return spconv._as_i32(coords), seed, ready

    def forward(self, batch_dict):
        """Static mode ('virconv_static': executor.StaticSpec): capacity-sized inputs + device row count, projection block
        already on the device ('virconv_proj', [B,28], ops.projection_params) — nothing reads a device value or uploads from
        pageable memory, so the call can be captured into a CUDA graph."""
        rot_num = batch_dict['transform_param'].shape[1] if 'transform_param' in batch_dict else 1
        ops.stats_arena(batch_dict['voxel_features'].device).reset()    # one memset for all BN accumulators of this pass
        for i in range(rot_num):
            rid = '' if i == 0 else str(i)
            feats = batch_dict['voxel_features' + rid]
            feats[:, 4:7] = 0                                    # RGB channels unused (:636), in place like the reference
            *xs, out = self._nrconv_stream(batch_dict, self._plan(), feats, batch_dict['voxel_coords' + rid],
                                           _copy_transform(batch_dict, i), rid, '', proj=batch_dict.get('virconv_proj'),
                                           static=batch_dict.get('virconv_static'), out=self.conv_out)
            _publish(batch_dict, rid, xs, out)
        return batch_dict


def _module_path_under_determinism(reason):
    """torch.use_deterministic_algorithms(True) and a forward that takes the per-operator module path, whose scatter
    dgrads, weight gradients and BatchNorm sums use float atomics: torch's contract for an operation without a
    deterministic implementation — raise, or warn under warn_only=True."""
    if not torch.are_deterministic_algorithms_enabled():
        return
    msg = ('VirConv backbone: the per-operator module path (%s) has no deterministic implementation; the plan executor '
           'has one' % reason)
    if torch.is_deterministic_algorithms_warn_only_enabled():
        warnings.warn(msg)
    else:
        raise RuntimeError(msg)


# module-path reasons that depend on one rank's batch or call rather than on the model or the configuration
NO_VOXELS, GRAD_INTO_FEATURES = 'no input voxels', 'gradient into the voxel features'
MIXED_MODES = 'BatchNorm layers in mixed train / eval modes'
_RANK_DEPENDENT = (NO_VOXELS, GRAD_INTO_FEATURES, MIXED_MODES)


def _module_path_reason(feats, plan=None, discard=False):
    """None when a forward over `feats` may run through the executor `plan`, else why it takes the per-operator module path.
    discard: it applies host-drawn or caller-given StVD kept rows.  Without a plan (a caller that only knows the plan did
    not run) the last reason is assumed."""
    if not executor.ENABLED:
        return 'VIRCONV_EXECUTOR=0'
    if not feats.is_cuda:
        return 'features not on a CUDA device'
    if feats.shape[0] == 0:
        return NO_VOXELS
    if feats.requires_grad:          # (the plan does not propagate a gradient into the voxel features; the module path does)
        return GRAD_INTO_FEATURES
    if discard:
        return 'host-drawn or caller-given StVD layer discard'
    if plan is not None and not plan.eligible():    # (dtype / layout / module type may change under .half(), .to())
        return 'SyncBatchNorm on mixed process groups, momentum=None, bias or a non-fp32 module'
    if plan is None or any(bn.training != plan.layers[0][1].training for _, bn in plan.layers):
        return MIXED_MODES
    return None


def decompose_tensor(t, i, batch_size):
    """Split the i-th transformed copy back out of an x-axis-batched tensor (spconv_backbone.py:314-337):
    rows with `i*q < x < (i+1)*q` (strict on both sides — the reference drops the x == i*q column), q = W // 4."""
    q = t.spatial_shape[2] // 4
    idx = spconv._as_i32(t.indices)
    x = idx[:, 3]
    rows = torch.nonzero((x > i * q) & (x < (i + 1) * q)).squeeze(1).to(torch.int32)   # data-dependent size (eval only)
    feats = ops.gather_rows(t.features, rows)
    sub = ops.gather_rows(idx, rows)
    sub[:, 3] -= i * q
    return spconv.SparseConvTensor(feats, sub, [t.spatial_shape[0], t.spatial_shape[1], q], batch_size)


class EvalStaticSpec:
    """Static (CUDA-graph capturable) test-time forward of VirConv8x over R = 1..4 transformed copies, given as
    batch_dict['virconv_eval_static'] (graph.GraphedForward builds one per capture).  The copies' inputs are the capacity-sized
    'voxel_features{i}' / 'voxel_coords{i}' (LiDAR, int32 coordinates) and 'voxel_features_mm{i}' / 'voxel_coords_mm{i}'
    (virtual points), i = '', '1', '2', ... as the reference suffixes them.
      lidar        executor.StaticSpec of the x-batched LiDAR plan over [D, H, 4W]; its n_dev receives the packed row count
                   (ops.xbatch_pack writes it on the device);
      lidar_counts R device int32[1]: the valid rows of each LiDAR copy;
      mm           R executor.StaticSpecs, one per copy of the virtual-point stream (n_dev: that copy's valid rows);
      proj         [R, B, 28] device projection blocks (ops.projection_params of each copy's transform)."""

    def __init__(self, lidar, lidar_counts, mm=(), proj=None):
        self.lidar, self.lidar_counts, self.mm, self.proj = lidar, list(lidar_counts), list(mm), proj

    @property
    def rot_num(self):
        return len(self.lidar_counts)


class VirConv8x(_VirConvBackbone):
    """VirConv-T / VirConv-S backbone (spconv_backbone.py:232-535): a LiDAR stream whose submanifold convs share one
    rulebook per stage (indice_keys 'subm1'..'subm4') plus, when `MM`, the virtual-point stream of NRConv blocks.
    Eval mode batches the ROT_NUM transformed copies along x into one [D, H, 4W] tensor (:360,:418-432) and splits the
    published tensors afterwards.

    Static mode (CUDA-graph capturable training forward, graph.GraphedStep): each stream takes its own executor.StaticSpec —
    batch_dict['virconv_static'] for the LiDAR stream, batch_dict['virconv_static_mm'] for the virtual-point stream, whose
    inputs are then capacity sized — and the MM stream reads the shared projection block batch_dict['virconv_proj'] ([B,28]
    on the device).  The nine published tensors follow VirConvL8x's static contract (capacity-sized features with a zero
    tail, indices with a -1 tail, device int32 `.num_rows`), as do the device-drawn StVD lists in 'stvd_kept_rows'.  The eval
    forward raises ValueError when given those training StaticSpecs; its static form (graph.GraphedForward) takes an
    EvalStaticSpec in batch_dict['virconv_eval_static']: ops.xbatch_pack -> the LiDAR plan over [D, H, 4W] ->
    ops.xbatch_split of x_conv3, x_conv4 and out, and one static run of the virtual-point plan per copy."""

    _input_discard = True

    def __init__(self, model_cfg, input_channels, grid_size, discard_mode='spconv2_compat', precision='fp32',
                 discard_rng='numpy', **kwargs):
        super().__init__(model_cfg, grid_size, discard_mode, discard_rng)
        f = self.num_filters
        self.mm = bool(_cfg_get(model_cfg, 'MM', False))
        self.conv_input = spconv.SparseSequential(
            spconv.SubMConv3d(input_channels, f[0], 3, padding=1, bias=False, indice_key='subm1'), norm_fn(f[0]), nn.ReLU())
        sub = lambda ci, co, key: sparse_block(ci, co, 3, norm_fn, 3, 'subm', padding=1, indice_key=key)
        down = lambda ci, co, key, pad: sparse_block(ci, co, 3, norm_fn, 3, 'spconv', stride=2, padding=pad, indice_key=key)
        self.conv1 = spconv.SparseSequential(sub(f[0], f[0], 'subm1'))
        self.conv2 = spconv.SparseSequential(down(f[0], f[1], 'spconv2', 1), sub(f[1], f[1], 'subm2'), sub(f[1], f[1], 'subm2'))
        self.conv3 = spconv.SparseSequential(down(f[1], f[2], 'spconv3', 1), sub(f[2], f[2], 'subm3'), sub(f[2], f[2], 'subm3'))
        self.conv4 = spconv.SparseSequential(down(f[2], f[3], 'spconv4', (0, 1, 1)), sub(f[3], f[3], 'subm4'),
                                             sub(f[3], f[3], 'subm4'))
        self._add_conv_out()
        if self.mm:
            self._add_nrconv_blocks(input_channels)
        spconv.set_precision(self, precision)

    # -- native plans (csrc/executor.cu) -----------------------------------------------------------------------
    def _plan_lidar(self):
        """LiDAR stream (:248-291): the submanifold convs of a stage share one rulebook ('subm1'..'subm4')."""
        def build():
            plan = executor.Plan(self.conv_input[0].in_channels)
            c0 = self.conv_input[0]
            rb = plan.subm_rb(0, 3, c0.kernel_size, c0.dilation, unique=True, keys=[c0.indice_key])
            f = plan.cbr(0, rb, c0, self.conv_input[1], seq=self.conv_input)
            f = plan.cbr(f, rb, self.conv1[0][0], self.conv1[0][1], seq=self.conv1[0])
            iset = 0
            plan.publish('x_conv1', f, iset)
            for name, stage in (('x_conv2', self.conv2), ('x_conv3', self.conv3), ('x_conv4', self.conv4)):
                down = stage[0][0]
                iset, rbd = plan.conv_rb(iset, 3, down.kernel_size, down.stride, down.padding, down.dilation,
                                         keys=[down.indice_key])
                c1 = stage[1][0]
                rb = plan.subm_rb(iset, 3, c1.kernel_size, c1.dilation, unique=True, keys=[c1.indice_key])
                f = plan.cbr(f, rbd, down, stage[0][1], seq=stage[0])
                f = plan.cbr(f, rb, c1, stage[1][1], seq=stage[1])
                f = plan.cbr(f, rb, stage[2][0], stage[2][1], seq=stage[2])
                plan.publish(name, f, iset)
            return self._plan_conv_out(plan, f, iset)
        return self._cached_plan('_plan_lidar_cache', build)

    def _plan_mm(self, stvd=False):
        """Virtual-point stream (:468-535).  stvd: with the device-drawn layer discards at sites 0 (the input voxels, :489)
        and 1-3 (after vir_conv1..3); the LiDAR stream has none in the reference."""
        return self._cached_plan('_plan_mm_stvd_cache' if stvd else '_plan_mm_cache', lambda: self._nrconv_plan(stvd)[0])

    @property
    def static_streams(self):
        """Batch-key suffixes of the input streams of a static-mode training forward: '' = the LiDAR stream
        ('voxel_features', 'voxel_coords', 'virconv_static'), '_mm' = the virtual-point stream ('voxel_features_mm',
        'voxel_coords_mm', 'virconv_static_mm')."""
        return ('', '_mm') if self.mm else ('',)

    def _check_static(self, batch_dict, rot_num):
        """Static mode (one executor.StaticSpec per stream) covers what runs through the plan executor in a training forward;
        anything else would silently compute over capacity-sized buffers as if every row were valid."""
        given = [s for s in ('', '_mm') if batch_dict.get('virconv_static' + s) is not None]
        if not given:
            return False
        if not self.training:
            raise ValueError('VirConv8x: static mode covers the training forward only — the eval forward batches the ROT_NUM '
                             'copies along x and splits the published tensors with data-dependent row counts (decompose_tensor)')
        if rot_num != 1:
            raise ValueError('VirConv8x: static mode takes one copy per stream (no transform_param)')
        if set(given) != set(self.static_streams):
            raise ValueError('VirConv8x: static mode needs a StaticSpec for each stream: %s'
                             % ', '.join("batch_dict['virconv_static%s']" % s for s in self.static_streams))
        if any(batch_dict['virconv_static' + s].phase != 0 for s in given):
            raise ValueError('VirConv8x: phased static execution (graph.PipelinedStep) covers VirConvL8x only')
        if self.mm:
            if batch_dict.get('virconv_proj') is None:
                raise ValueError("VirConv8x: static mode needs batch_dict['virconv_proj'] (ops.projection_params on the device)")
            if self._host_discard(batch_dict):
                raise ValueError("VirConv8x: static mode runs the StVD layer discard in the plan (discard_rng='device'); "
                                 'host-drawn or caller-given kept rows have no static form')
        return True

    def _check_eval_static(self, batch_dict, rot_num):
        """-> the EvalStaticSpec of a static test-time forward, or None.  (Runs after _check_static: given the training specs
        too, an eval forward raises their refusal first.)"""
        spec = batch_dict.get('virconv_eval_static')
        if spec is None:
            return None
        if self.training:
            raise ValueError("VirConv8x: batch_dict['virconv_eval_static'] is the test-time forward (model.eval()); a static "
                             "training forward takes virconv_static / virconv_static_mm (graph.GraphedStep)")
        if not 1 <= rot_num <= ops.XBATCH_MAX:
            raise ValueError('VirConv8x: the x-batched eval forward takes 1..%d transformed copies (the factor 4 of the [D, H, 4W] '
                             'grid is fixed, spconv_backbone.py:360); transform_param has %d' % (ops.XBATCH_MAX, rot_num))
        if spec.rot_num != rot_num or (self.mm and len(spec.mm) != rot_num):
            raise ValueError('VirConv8x: the EvalStaticSpec describes %d LiDAR / %d virtual-point copies, transform_param %d'
                             % (spec.rot_num, len(spec.mm), rot_num))
        if spec.lidar is None or (self.mm and (spec.proj is None or tuple(spec.proj.shape[:2]) != (rot_num, batch_dict['batch_size']))):
            raise ValueError('VirConv8x: the EvalStaticSpec needs the packed LiDAR StaticSpec and [R, B, 28] projection blocks')
        sfx = [''] + [str(i) for i in range(1, rot_num)]
        keys = [k + s for s in sfx for k in ('voxel_features', 'voxel_coords')]
        if self.mm:
            keys += [k + '_mm' + s for s in sfx for k in ('voxel_features', 'voxel_coords')]
        missing = [k for k in keys if batch_dict.get(k) is None]
        if missing:
            raise ValueError('VirConv8x static eval forward: the batch has no %s' % ', '.join(missing))
        return spec

    def _eval_static_forward(self, batch_dict, spec, sfx, batch_size):
        """The eval forward below with every row count on the device (see EvalStaticSpec)."""
        R = len(sfx)
        feats = [batch_dict['voxel_features' + s] for s in sfx]
        coords = [spconv._as_i32(batch_dict['voxel_coords' + s]) for s in sfx]
        pf, pc, _ = ops.xbatch_pack(feats, coords, spec.lidar_counts, self.sparse_shape[2], spec.lidar.n_dev)
        big = [self.sparse_shape[0], self.sparse_shape[1], self.sparse_shape[2] * 4]      # factor 4 is hard-coded (:360)
        _, _, x3, x4, out = self._lidar_stream(pf, pc, big, batch_size, static=spec.lidar)

        def split(t):
            q = t.spatial_shape[2] // 4
            parts = []
            for f, idx, n in ops.xbatch_split(t.features, spconv._as_i32(t.indices), t.num_rows, t.spatial_shape[2], R):
                p = spconv.SparseConvTensor(f, idx, [t.spatial_shape[0], t.spatial_shape[1], q], batch_size)
                p.num_rows = n
                parts.append(p)
            return parts

        x3s, x4s, outs = split(x3), split(x4), split(out)
        for i, s in enumerate(sfx):
            _publish(batch_dict, s, (None, None, x3s[i], x4s[i]), outs[i])
        if not self.mm:
            return batch_dict
        plan = self._plan_mm()
        for i, s in enumerate(sfx):
            xs = self._nrconv_stream(batch_dict, plan, batch_dict['voxel_features_mm' + s], batch_dict['voxel_coords_mm' + s],
                                     None, s, '_mm' + s, proj=spec.proj[i], static=spec.mm[i],
                                     refusal='VirConv8x static eval forward: the virtual-point stream cannot run through the '
                                             'plan executor (%s)')
            _publish(batch_dict, s, xs, stream='_mm')
        return batch_dict

    def _lidar_stream(self, feats, coords, shape, batch_size, static=None):
        plan = self._plan_lidar()
        reason = _module_path_reason(feats, plan)
        if reason is None:
            return self._run(plan, feats, coords, shape, batch_size, None, '', static=static)[1]
        if static is not None:
            raise ValueError('VirConv8x static mode: the LiDAR stream cannot run through the plan executor (%s)' % reason)
        self._no_module_path_under_sync(plan, reason)
        _module_path_under_determinism(reason)
        x = spconv.SparseConvTensor(feats, coords.int(), shape, batch_size)
        x1 = self.conv1(self.conv_input(x))
        x2 = self.conv2(x1)
        x3 = self.conv3(x2)
        x4 = self.conv4(x3)
        return x1, x2, x3, x4, self.conv_out(x4)

    def forward(self, batch_dict):
        rot_num = batch_dict['transform_param'].shape[1] if 'transform_param' in batch_dict else 1
        batch_size = batch_dict['batch_size']
        sfx = [''] + [str(i) for i in range(1, rot_num)]
        static = self._check_static(batch_dict, rot_num)
        eval_static = self._check_eval_static(batch_dict, rot_num)
        ops.stats_arena(batch_dict['voxel_features'].device).reset()
        if eval_static is not None:
            return self._eval_static_forward(batch_dict, eval_static, sfx, batch_size)
        if self.training:
            for s in sfx:
                *xs, out = self._lidar_stream(batch_dict['voxel_features' + s], batch_dict['voxel_coords' + s],
                                              self.sparse_shape, batch_size, batch_dict.get('virconv_static'))
                _publish(batch_dict, s, xs, out)
        else:
            feats, coords = [], []
            for i, s in enumerate(sfx):
                feats.append(batch_dict['voxel_features' + s])
                c = batch_dict['voxel_coords' + s].clone()
                c[:, 3] += i * self.sparse_shape[2]
                coords.append(c)
            big = [self.sparse_shape[0], self.sparse_shape[1], self.sparse_shape[2] * 4]      # factor 4 is hard-coded (:360)
            _, _, x3, x4, out = self._lidar_stream(torch.cat(feats, 0), torch.cat(coords), big, batch_size)
            for i, s in enumerate(sfx):
                out_i = decompose_tensor(out, i, batch_size)
                _publish(batch_dict, s, (None, None, decompose_tensor(x3, i, batch_size), decompose_tensor(x4, i, batch_size)),
                         out_i)
        if self.mm:
            for i, s in enumerate(sfx):
                # static mode: the shared projection block is already on the device ('virconv_proj', [B,28])
                xs = self._nrconv_stream(
                    batch_dict, self._plan_mm(self._device_discard()), batch_dict['voxel_features_mm' + s],
                    batch_dict['voxel_coords_mm' + s], _copy_transform(batch_dict, i), s, '_mm' + s,
                    proj=batch_dict['virconv_proj'] if static else None, static=batch_dict.get('virconv_static_mm'),
                    refusal='VirConv8x static mode: the virtual-point stream cannot run through the plan executor (%s)'
                    if static else None)
                _publish(batch_dict, s, xs, stream='_mm')
        return batch_dict
