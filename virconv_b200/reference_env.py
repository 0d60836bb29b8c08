"""Make the reference's OWN Python (`pcdet/`, `tools/train.py`, `tools/test.py`) importable on this stack (Python 3.12, torch
2.11, no spconv / cumm / compiled `pcdet.ops` extensions) — SURVEY §8f-2.

    import virconv_b200.reference_env as renv
    renv.install(use_fused_backbones=True)      # before anything from `pcdet` is imported

What it registers (nothing is written into the reference tree, nothing from it is copied):
  * `spconv`, `spconv.pytorch`, `spconv.utils`, `cumm.tensorview`      -> virconv_b200.spconv_compat (the sm_90a kernels)
  * Python-3.12 compatibility: `collections.Iterable` & friends (tools/train_utils/optimization/fastai_optim.py:3),
    `numpy.int/float/bool` aliases the 2021-era code still uses
  * small pure-Python stand-ins when the real package is absent: `easydict.EasyDict`, `tensorboardX.SummaryWriter`
    (falls back to a no-op writer), `prefetch_generator.BackgroundGenerator`, `skimage.transform` (import only)
  * the six compiled extensions of `pcdet/ops` (setup.py:52-128) as Python modules:
      - `pointnet2_stack_cuda.voxel_query_wrapper / group_points_wrapper / group_points_grad_wrapper` run on this
        library's kernels (vc_voxel_query, vc_group_points, vc_group_points_grad: bit-exact against the reference's own
        CUDA, tests/test_gpu_roi_pool.py) — the voxel-RoI pooling of TEDMHead (ted_head.py:496-552);
      - `iou3d_nms_cuda.boxes_overlap_bev_gpu / boxes_iou_bev_gpu / nms_gpu / nms_normal_gpu / boxes_iou_bev_cpu` run
        on this library's rotated-box kernels (csrc/iou3d_nms.cu; the CPU one on its host entry point), with the
        pybind signatures of iou3d_nms_api.cpp: the proposal / final NMS, RoI target assignment and GT sampling;
      - `roiaware_pool3d_cuda.points_in_boxes_cpu` (dataset-side augmentation) is restated in torch;
      - everything else (ball query, FPS, points_in_boxes_gpu, RoI-point pooling, deformable conv, VOTR ops) is
        import-only: calling it raises NotImplementedError naming the reference source that would have to be built.
With `use_fused_backbones` the detector registry (`pcdet.models.backbones_3d.__all__`) hands out this package's
VirConvL8x / VirConv8x (plan executor, fused conv+BN+ReLU) instead of the reference classes over the compat layer.
With `use_fused_roi_pool` `pcdet.ops.pointnet2.pointnet2_stack.voxel_pool_modules.NeighborVoxelSAModuleMSG` is this
package's fused class (virconv_b200.voxel_pool), so TEDMHead's RoI grid pooling layers are built from it unchanged.
With `use_fused_rpn_targets` `AnchorHeadSingle.get_anchor_mask` and the `AxisAlignedTargetAssigner` the anchor heads build
(looked up in anchor_head_template, which imports the name at module level, and in its own module) are this package's
device versions (virconv_b200.anchor_targets): the RPN's anchor mask and target assignment without a host read.
With `use_fused_roi_targets` the `ProposalTargetLayer` the RoI heads build (looked up in roi_head_template, which imports
the name at module level, and in its own module) and `RoIHeadTemplate.assign_targets` are this package's device versions
(virconv_b200.roi_targets): the RCNN's RoI sampling, labels and canonical transform in one call without a host read.
With `use_fused_losses` `AnchorHeadTemplate.get_loss` and `RoIHeadTemplate.get_loss` are this package's drop-in methods
(virconv_b200.head_losses): the RPN and RCNN training losses and their gradients in one kernel call each, without a host
read apart from the one copy of the tb values.
With `use_fused_part_pool` `TEDMHead.obtain_conf_preds` is this package's drop-in method (virconv_b200.part_pool): the
PART branch's position-sensitive RoI pooling of VirConv-T / -S in one call per stage, without a host read, with a
bit-reproducible part-map gradient.
With `use_fused_roi_grid` `TEDMHead.roi_grid_pool` and `roi_grid_pool_mm` are this package's drop-in methods
(virconv_b200.roi_grid): the grid points and their voxel coordinates in one launch per call, and the voxel -> row map and
voxel centres of each published tensor built once per forward, without a host read.
With `use_fused_box_decode` `AnchorHeadTemplate.generate_predicted_boxes`, `RoIHeadTemplate.generate_predicted_boxes` and
`TEDMHead.roi_x_trans / roi_score_trans / pred_x_trans` are this package's drop-in methods (virconv_b200.box_decode): the
heads' box decoding and the cascade stage transforms in one launch per call, with transform_param read on the device.
With `use_fused_kitti_eval` `get_official_eval_result`, `get_coco_eval_result` and the imported name `rotate_iou_gpu_eval`
of kitti_object_eval_python.eval are this package's (virconv_b200.kitti_eval): KittiDatasetMM.evaluation, which imports
the module inside the method, then runs the KITTI evaluation in nine launches with one upload and one read-back.
With `use_fused_optimizer` `train_utils.optimization.build_optimizer` (tools/train_utils/optimization/__init__.py:11-36, the
name tools/train.py imports with tools/ on sys.path) returns this package's optim.FusedAdamOneCycle for OPTIMIZER
adam_onecycle / adam_cosin and calls the reference's function for every other value, and the `clip_grad_norm_` name
`train_utils.train_utils` imported at module level records its max_norm for the next step() of the fused optimizer that
owns those parameters, leaving the gradients alone (parameters no fused optimizer owns go to torch's function): the
reference's train_one_epoch (train_utils.py:13-71) then runs unchanged, with clipping, decay and Adam in two launches.
With `use_device_input_discard` `DatasetTemplate.input_point_discard` returns its input, `DataProcessor.shuffle_points` passes
the frame through and `DataProcessor.mask_points_and_boxes_outside_range` filters the boxes only: `prepare_data` then hands
over the split but undiscarded, unmasked, unshuffled cloud, and the model side runs the StVD input front end on the device
(preprocess.input_front_end, or GraphedStep's voxelizer entry `input_discard`).  The points mask has to move with the
discard: the reference bins the virtual points before the range mask, so masking them first would change every `out_n`.
"""
from __future__ import annotations

import collections
import functools
import collections.abc
import importlib
import sys
import types

import numpy as np
import torch


class EasyDict(dict):
    """Attribute-style dict, nested (what `pcdet/config.py` needs from the `easydict` package)."""

    def __init__(self, d=None, **kwargs):
        super().__init__()
        d = dict(d or {})
        d.update(kwargs)
        for k, v in d.items():
            setattr(self, k, v)

    def __setattr__(self, name, value):
        if isinstance(value, (list, tuple)):
            value = type(value)(EasyDict(x) if isinstance(x, dict) and not isinstance(x, EasyDict) else x for x in value)
        elif isinstance(value, dict) and not isinstance(value, EasyDict):
            value = EasyDict(value)
        super().__setattr__(name, value)
        super().__setitem__(name, value)

    __setitem__ = __setattr__

    def update(self, e=None, **f):
        d = dict(e or {})
        d.update(f)
        for k, v in d.items():
            setattr(self, k, v)

    def pop(self, k, *a):
        if hasattr(self, k):
            delattr(self, k)
        return super().pop(k, *a)


class _NullWriter:
    def __init__(self, *a, **k):
        pass

    def __getattr__(self, name):
        return lambda *a, **k: None


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__path__ = []
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def _missing(name):
    try:
        importlib.import_module(name)
        return False
    except Exception:       # noqa: BLE001
        return True


def _unbuilt(ext, fn, src):
    def f(*a, **k):
        raise NotImplementedError(f'{ext}.{fn}: this compiled extension of the reference ({src}) is not on the VirConv sparse-conv '
                                  f'hot path and has no sm_90a build in virconv_b200 (SURVEY §2b / §8f-2)')
    f.__name__ = fn
    return f


def _stub_ext(modname, src, fns, **real):
    attrs = {fn: _unbuilt(modname.rsplit('.', 1)[-1], fn, src) for fn in fns}
    attrs.update(real)
    m = types.ModuleType(modname)
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[modname] = m
    parent, leaf = modname.rsplit('.', 1)
    if parent in sys.modules:
        setattr(sys.modules[parent], leaf, m)
    return m


# ---- pointnet2_stack: the voxel-RoI pooling primitives, on this library's kernels ---------------------------------------
def _voxel_query_wrapper(M, R1, R2, R3, nsample, radius, z_range, y_range, x_range, new_xyz, xyz, new_coords, point_indices, idx):
    """pointnet2_stack_cuda.voxel_query_wrapper (voxel_query_utils.py:30-33): writes idx [M, nsample] in place."""
    from . import _lib, ops
    lib = _lib.load()
    _lib.check(lib.vc_voxel_query(int(M), int(R1), int(R2), int(R3), int(nsample), float(radius), int(z_range), int(y_range),
                                  int(x_range), ops._p(new_xyz), ops._p(xyz), ops._p(new_coords), ops._p(point_indices),
                                  ops._p(idx), None, ops._stream()), 'vc_voxel_query')


def _group_points_wrapper(B, M, C, nsample, features, features_batch_cnt, idx, idx_batch_cnt, out):
    """pointnet2_stack_cuda.group_points_wrapper (pointnet2_utils.py:74-75): out [M, C, nsample]."""
    from . import _lib, ops
    lib = _lib.load()
    _lib.check(lib.vc_group_points(int(B), int(M), int(C), int(nsample), ops._p(features), ops._p(features_batch_cnt), ops._p(idx),
                                   ops._p(idx_batch_cnt), ops._p(out), ops._stream()), 'vc_group_points')


def _group_points_grad_wrapper(B, M, C, N, nsample, grad_out, idx, idx_batch_cnt, features_batch_cnt, grad_features):
    """pointnet2_stack_cuda.group_points_grad_wrapper (pointnet2_utils.py:95-96): grad_features [N, C] (zeroed by the caller)."""
    from . import _lib, ops
    lib = _lib.load()
    _lib.check(lib.vc_group_points_grad(int(B), int(M), int(C), int(N), int(nsample), ops._p(grad_out), ops._p(idx),
                                        ops._p(idx_batch_cnt), ops._p(features_batch_cnt), ops._p(grad_features), ops._stream()),
               'vc_group_points_grad')


# ---- iou3d_nms: rotated-box IoU / NMS, on this library's kernels (iou3d_nms_api.cpp:8-14) -------------------------------
def _pairwise_into(fn, boxes_a, boxes_b, out):
    from . import _lib, ops
    lib = _lib.load()
    ops._require_cuda(boxes_a, boxes_b, out)
    assert out.is_contiguous() and out.dtype == torch.float32
    a, b = boxes_a.contiguous(), boxes_b.contiguous()
    _lib.check(getattr(lib, fn)(a.data_ptr(), a.shape[0], b.data_ptr(), b.shape[0], out.data_ptr(), ops._stream()), fn)
    return 1


def _boxes_overlap_bev_gpu(boxes_a, boxes_b, ans_overlap):
    """iou3d_nms_cuda.boxes_overlap_bev_gpu (iou3d_nms.cpp:49-68): fills ans_overlap [N, M] with the BEV intersection areas."""
    return _pairwise_into('vc_boxes_overlap_bev', boxes_a, boxes_b, ans_overlap)


def _boxes_iou_bev_gpu(boxes_a, boxes_b, ans_iou):
    """iou3d_nms_cuda.boxes_iou_bev_gpu (iou3d_nms.cpp:70-88): fills ans_iou [N, M] with the BEV IoU."""
    return _pairwise_into('vc_boxes_iou_bev', boxes_a, boxes_b, ans_iou)


def _boxes_iou_bev_cpu(boxes_a, boxes_b, ans_iou):
    """iou3d_nms_cuda.boxes_iou_bev_cpu (iou3d_cpu.cpp:232-252): CPU tensors, fills ans_iou [N, M]."""
    from . import _lib
    assert not (boxes_a.is_cuda or boxes_b.is_cuda or ans_iou.is_cuda), 'Only support CPU tensors'
    assert ans_iou.is_contiguous() and ans_iou.dtype == torch.float32
    a, b = boxes_a.float().contiguous(), boxes_b.float().contiguous()
    _lib.check(_lib.load().vc_boxes_iou_bev_host(a.data_ptr(), a.shape[0], b.data_ptr(), b.shape[0], ans_iou.data_ptr()),
               'vc_boxes_iou_bev_host')
    return 1


def _nms_into(boxes, keep, thresh, normal):
    from . import iou3d_nms
    n = boxes.shape[0]
    if n == 0:
        return 0
    counts = torch.full((1,), n, dtype=torch.int32, device=boxes.device)
    k, num = iou3d_nms._nms_sorted(boxes.float().contiguous().view(1, n, -1), counts, thresh, n, normal)
    num_out = int(num.item())
    keep[:num_out] = k[0, :num_out].cpu().to(keep.dtype)
    return num_out


def _nms_gpu(boxes, keep, nms_overlap_thresh):
    """iou3d_nms_cuda.nms_gpu (iou3d_nms.cpp:90-136): boxes [N, 7] on the GPU, already in descending score order; writes the
    kept row indices into the CPU LongTensor `keep` and returns their number."""
    return _nms_into(boxes, keep, nms_overlap_thresh, False)


def _nms_normal_gpu(boxes, keep, nms_overlap_thresh):
    """iou3d_nms_cuda.nms_normal_gpu (iou3d_nms.cpp:139-186): the axis-aligned variant of _nms_gpu."""
    return _nms_into(boxes, keep, nms_overlap_thresh, True)


def _points_in_boxes_cpu(boxes, points, point_indices):
    """roiaware_pool3d_cuda.points_in_boxes_cpu (roiaware_pool3d_utils.py:9-26; src/roiaware_pool3d.cpp:106-140): CPU tensors,
    boxes [N, 7] (x, y, z, dx, dy, dz, heading) with z at the box centre, points [M, 3]; point_indices [N, M] int32 set to 1
    where the point lies inside the box (|local z| <= dz/2, |local x| < dx/2, |local y| < dy/2 after rotating by -heading)."""
    b = boxes.float()
    p = points.float()
    dz = (p[None, :, 2] - b[:, None, 2]).abs()
    sx, sy = p[None, :, 0] - b[:, None, 0], p[None, :, 1] - b[:, None, 1]
    c, s = torch.cos(-b[:, 6])[:, None], torch.sin(-b[:, 6])[:, None]
    lx = sx * c - sy * s
    ly = sx * s + sy * c
    inside = (dz <= b[:, None, 5] / 2) & (lx.abs() < b[:, None, 3] / 2) & (ly.abs() < b[:, None, 4] / 2)
    point_indices.copy_(inside.to(point_indices.dtype))
    return 1


def _fused_build_optimizer(reference_build):
    def build_optimizer(model, optim_cfg):
        """build_optimizer (optimization/__init__.py:11-36) with the adam_onecycle / adam_cosin branch on vc_optim_step."""
        if optim_cfg.OPTIMIZER not in ('adam_onecycle', 'adam_cosin'):
            return reference_build(model, optim_cfg)
        from .optim import FusedAdamOneCycle
        return FusedAdamOneCycle.from_model(model, wd=optim_cfg.WEIGHT_DECAY, lr=3e-3, betas=(0.9, 0.99))
    build_optimizer._reference = reference_build
    return build_optimizer


def _fused_clip_grad_norm_(parameters, max_norm, *args, **kwargs):
    """clip_grad_norm_ as train_utils.py:50 calls it: the fused optimizers owning `parameters` clip inside their next step();
    what is left goes to torch's function.  -> None or torch's result for the rest (train_one_epoch ignores it)."""
    from . import optim
    params = [parameters] if isinstance(parameters, torch.Tensor) else list(parameters)
    ids = {id(p) for p in params}
    for opt in optim.live_optimizers():
        own = opt.owns(ids)
        if own:
            opt.clip_grad_norm(max_norm)
            ids -= own
    rest = [p for p in params if id(p) in ids and p.grad is not None]
    return torch.nn.utils.clip_grad_norm_(rest, max_norm, *args, **kwargs) if rest else None


def _keep_points(self, points, bin_num=2, rate=0.8):
    """`DatasetTemplate.input_point_discard` under `use_device_input_discard`: the virtual points pass unchanged."""
    return points


def _shuffle_later(self, data_dict=None, config=None):
    """`DataProcessor.shuffle_points` under `use_device_input_discard`: the order is drawn on the device."""
    if data_dict is None:
        return functools.partial(self.shuffle_points, config=config)
    return data_dict


def _mask_boxes_only(self, data_dict=None, config=None):
    """`DataProcessor.mask_points_and_boxes_outside_range` under `use_device_input_discard`: the boxes of every copy are
    filtered as before (REMOVE_OUTSIDE_BOXES, min_num_corners), the points are left for the device front end, which masks
    them after its discard."""
    if data_dict is None:
        return functools.partial(self.mask_points_and_boxes_outside_range, config=config)
    if not config.REMOVE_OUTSIDE_BOXES:
        return data_dict
    box_utils = importlib.import_module('pcdet.utils.box_utils')
    for r in range(self.rot_num):
        key = 'gt_boxes' + (str(r) if r else '')
        boxes = data_dict.get(key)
        if boxes is None:
            continue
        inside = box_utils.mask_boxes_outside_range_numpy(boxes, self.point_cloud_range,
                                                          min_num_corners=config.get('min_num_corners', 1))
        data_dict[key] = boxes[inside]
        if r == 0 and 'gt_tracklets' in data_dict:
            data_dict['gt_tracklets'] = data_dict['gt_tracklets'][inside]
            data_dict['num_bbs_in_tracklets'] = data_dict['num_bbs_in_tracklets'][inside]
    return data_dict


def install(use_fused_backbones=False, reference_root=None, use_fused_roi_pool=False, use_fused_rpn_targets=False,
            use_fused_roi_targets=False, use_fused_losses=False, use_fused_part_pool=False, use_fused_optimizer=False, use_fused_roi_grid=False,
            use_fused_box_decode=False, use_fused_kitti_eval=False, use_device_input_discard=False):
    """Register everything listed in the module docstring.  `reference_root`: put that checkout first on sys.path."""
    if reference_root is not None and reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    from . import spconv_compat
    spconv_compat.install_as_spconv()
    # Python 3.10+: the ABC aliases left `collections`; numpy 1.24+: the builtin aliases left `numpy`
    for name in ('Iterable', 'Mapping', 'MutableMapping', 'Sequence', 'Callable'):
        if not hasattr(collections, name):
            setattr(collections, name, getattr(collections.abc, name))
    for name, typ in (('int', int), ('float', float), ('bool', bool), ('object', object)):
        if name not in np.__dict__:
            try:
                setattr(np, name, typ)
            except Exception:       # noqa: BLE001
                pass
    if _missing('easydict'):
        _module('easydict', EasyDict=EasyDict)
    if _missing('tensorboardX'):
        writer = _NullWriter
        try:
            from torch.utils.tensorboard import SummaryWriter as writer     # noqa: N813
        except Exception:       # noqa: BLE001
            pass
        _module('tensorboardX', SummaryWriter=writer)
    if _missing('prefetch_generator'):
        class BackgroundGenerator:
            def __init__(self, generator, max_prefetch=1):
                self._g = iter(generator)

            def __iter__(self):
                return self._g

            def __next__(self):
                return next(self._g)
        _module('prefetch_generator', BackgroundGenerator=BackgroundGenerator)
    if _missing('skimage'):
        sk = _module('skimage')
        sk.transform = _module('skimage.transform', resize=_unbuilt('skimage.transform', 'resize', 'scikit-image'))
        sk.io = _module('skimage.io', imread=_unbuilt('skimage.io', 'imread', 'scikit-image'))

    # the compiled extensions of pcdet/ops: module objects under the names the reference imports
    _stub_ext('pcdet.ops.iou3d_nms.iou3d_nms_cuda', 'pcdet/ops/iou3d_nms/src', [],
              boxes_overlap_bev_gpu=_boxes_overlap_bev_gpu, boxes_iou_bev_gpu=_boxes_iou_bev_gpu, nms_gpu=_nms_gpu,
              nms_normal_gpu=_nms_normal_gpu, boxes_iou_bev_cpu=_boxes_iou_bev_cpu)
    _stub_ext('pcdet.ops.roiaware_pool3d.roiaware_pool3d_cuda', 'pcdet/ops/roiaware_pool3d/src',
              ['forward', 'backward', 'points_in_boxes_gpu'], points_in_boxes_cpu=_points_in_boxes_cpu)
    _stub_ext('pcdet.ops.roipoint_pool3d.roipoint_pool3d_cuda', 'pcdet/ops/roipoint_pool3d/src', ['forward'])
    _stub_ext('pcdet.ops.pointnet2.pointnet2_batch.pointnet2_batch_cuda', 'pcdet/ops/pointnet2/pointnet2_batch/src',
              ['ball_query_wrapper', 'group_points_wrapper', 'group_points_grad_wrapper', 'gather_points_wrapper',
               'gather_points_grad_wrapper', 'furthest_point_sampling_wrapper', 'three_nn_wrapper', 'three_interpolate_wrapper',
               'three_interpolate_grad_wrapper'])
    _stub_ext('pcdet.ops.pointnet2.pointnet2_stack.pointnet2_stack_cuda', 'pcdet/ops/pointnet2/pointnet2_stack/src',
              ['ball_query_wrapper', 'furthest_point_sampling_wrapper', 'three_nn_wrapper', 'three_interpolate_wrapper',
               'three_interpolate_grad_wrapper', 'stack_furthest_point_sampling_wrapper', 'query_stacked_local_neighbor_idxs_wrapper_stack',
               'query_three_nn_by_stacked_local_idxs_wrapper_stack', 'vector_pool_wrapper', 'vector_pool_grad_wrapper'],
              voxel_query_wrapper=_voxel_query_wrapper, group_points_wrapper=_group_points_wrapper,
              group_points_grad_wrapper=_group_points_grad_wrapper)
    _stub_ext('pcdet.ops.votr_ops.votr_ops_cuda', 'pcdet/ops/votr_ops/src', [])
    _stub_ext('pcdet.ops.dcn.deform_conv_cuda', 'pcdet/ops/dcn/src', [])
    if use_fused_backbones:
        b3d = importlib.import_module('pcdet.models.backbones_3d')
        from .backbone import VirConv8x, VirConvL8x
        b3d.__all__['VirConvL8x'] = VirConvL8x
        b3d.__all__['VirConv8x'] = VirConv8x
    if use_fused_roi_pool:
        vpm = importlib.import_module('pcdet.ops.pointnet2.pointnet2_stack.voxel_pool_modules')
        from .voxel_pool import NeighborVoxelSAModuleMSG
        vpm.NeighborVoxelSAModuleMSG = NeighborVoxelSAModuleMSG
    if use_fused_rpn_targets:
        from . import anchor_targets
        for name in ('pcdet.models.dense_heads.target_assigner.axis_aligned_target_assigner',
                     'pcdet.models.dense_heads.anchor_head_template'):
            importlib.import_module(name).AxisAlignedTargetAssigner = anchor_targets.AxisAlignedTargetAssigner
        ahs = importlib.import_module('pcdet.models.dense_heads.anchor_head_single')
        ahs.AnchorHeadSingle.get_anchor_mask = anchor_targets.get_anchor_mask
    if use_fused_roi_targets:
        from . import roi_targets
        for name in ('pcdet.models.roi_heads.target_assigner.proposal_target_layer',
                     'pcdet.models.roi_heads.roi_head_template'):
            importlib.import_module(name).ProposalTargetLayer = roi_targets.ProposalTargetLayer
        rht = importlib.import_module('pcdet.models.roi_heads.roi_head_template').RoIHeadTemplate
        if rht.assign_targets is not roi_targets.assign_targets:
            roi_targets._reference_assign_targets = rht.assign_targets
        rht.assign_targets = roi_targets.assign_targets
    if use_fused_losses:
        from . import head_losses
        aht = importlib.import_module('pcdet.models.dense_heads.anchor_head_template').AnchorHeadTemplate
        aht.get_loss = head_losses.anchor_head_get_loss
        rht = importlib.import_module('pcdet.models.roi_heads.roi_head_template').RoIHeadTemplate
        rht.get_loss = head_losses.roi_head_get_loss
    if use_fused_part_pool:
        from . import part_pool
        ted = importlib.import_module('pcdet.models.roi_heads.ted_head').TEDMHead
        if ted.obtain_conf_preds is not part_pool.obtain_conf_preds:
            part_pool._reference_obtain_conf_preds = ted.obtain_conf_preds
        ted.obtain_conf_preds = part_pool.obtain_conf_preds
    if use_fused_roi_grid:
        from . import roi_grid
        ted = importlib.import_module('pcdet.models.roi_heads.ted_head').TEDMHead
        if ted.roi_grid_pool is not roi_grid.roi_grid_pool:
            roi_grid._reference_roi_grid_pool = ted.roi_grid_pool
        if ted.roi_grid_pool_mm is not roi_grid.roi_grid_pool_mm:
            roi_grid._reference_roi_grid_pool_mm = ted.roi_grid_pool_mm
        ted.roi_grid_pool = roi_grid.roi_grid_pool
        ted.roi_grid_pool_mm = roi_grid.roi_grid_pool_mm
    if use_fused_box_decode:
        from . import box_decode
        aht = importlib.import_module('pcdet.models.dense_heads.anchor_head_template').AnchorHeadTemplate
        rht = importlib.import_module('pcdet.models.roi_heads.roi_head_template').RoIHeadTemplate
        ted = importlib.import_module('pcdet.models.roi_heads.ted_head').TEDMHead
        for cls, name, fused, record in (
                (aht, 'generate_predicted_boxes', box_decode.anchor_generate_predicted_boxes,
                 '_reference_anchor_generate_predicted_boxes'),
                (rht, 'generate_predicted_boxes', box_decode.roi_generate_predicted_boxes,
                 '_reference_roi_generate_predicted_boxes'),
                (ted, 'roi_x_trans', box_decode.roi_x_trans, '_reference_roi_x_trans'),
                (ted, 'roi_score_trans', box_decode.roi_score_trans, '_reference_roi_score_trans'),
                (ted, 'pred_x_trans', box_decode.pred_x_trans, '_reference_pred_x_trans')):
            if getattr(cls, name) is not fused:
                setattr(box_decode, record, getattr(cls, name))
            setattr(cls, name, fused)
    if use_fused_kitti_eval:
        from . import kitti_eval
        ev = importlib.import_module('pcdet.datasets.kitti.kitti_object_eval_python.eval')
        ev.get_official_eval_result = kitti_eval.get_official_eval_result
        ev.get_coco_eval_result = kitti_eval.get_coco_eval_result
        ev.rotate_iou_gpu_eval = kitti_eval.rotate_iou_eval
    if use_device_input_discard:
        ds = importlib.import_module('pcdet.datasets.dataset').DatasetTemplate
        ds.input_point_discard = _keep_points
        dp = importlib.import_module('pcdet.datasets.processor.data_processor').DataProcessor
        dp.shuffle_points = _shuffle_later
        dp.mask_points_and_boxes_outside_range = _mask_boxes_only
    if use_fused_optimizer:
        import os
        tools = os.path.join(reference_root, 'tools') if reference_root is not None else None
        if tools is not None and tools not in sys.path:
            sys.path.append(tools)              # (tools/train.py runs from tools/: `from train_utils.optimization import ...`)
        om = importlib.import_module('train_utils.optimization')
        if not hasattr(om.build_optimizer, '_reference'):
            om.build_optimizer = _fused_build_optimizer(om.build_optimizer)
        importlib.import_module('train_utils.train_utils').clip_grad_norm_ = _fused_clip_grad_norm_
    return True
