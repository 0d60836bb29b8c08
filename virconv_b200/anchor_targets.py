"""Anchor-head targets of the RPN (`AnchorHeadSingle` of VirConv-L / -T / -S) on the sm_90a kernels of
csrc/anchor_targets.cu, which states the rules.

  * `anchor_mask`               = AnchorHeadSingle.get_anchor_mask (anchor_head_single.py:75-115), on the device;
  * `AxisAlignedTargetAssigner` = the reference class (axis_aligned_target_assigner.py), same constructor and
                                  `assign_targets` result, all scenes and anchor sets in one batched call;
  * `assign_targets_batched`    = the same into caller-owned buffers, for CUDA-graph capture.

Nothing reads the device on the host once the shapes are known.  Supported: POS_FRACTION < 0 (no random subsampling),
MATCH_HEIGHT False, USE_MULTIHEAD False, NORM_BY_NUM_EXAMPLES False, a 7-value ResidualCoder — what the VirConv YAMLs
use; anything else is rejected at construction: use the reference class for it."""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, ops
from ._lib import check, host_f32, host_i32

MAX_GT = 512        # VC_ANCHOR_MAX_GT: GT rows per scene (padded count)
MAX_SETS = 8        # VC_ANCHOR_MAX_SETS
MAX_NAMES = 32      # VC_ANCHOR_MAX_NAMES
_REF = 'pcdet.models.dense_heads.target_assigner.axis_aligned_target_assigner.AxisAlignedTargetAssigner (the reference class)'


def mask_params(point_cloud_range, grid_size):
    """(min_x, min_y, 1/stride) as get_anchor_mask computes them on the GPU: stride = round(voxel_size * 8 * 10) with
    voxel_size = (range[3] - range[0]) / grid_size[0] in numpy's arithmetic, divided as torch's multiply by the fp32
    reciprocal"""
    pcr = np.asarray(point_cloud_range)
    voxel_size = (pcr[3] - pcr[0]) / np.asarray(grid_size)[0]
    stride = np.round(voxel_size * 8. * 10.)
    return np.float32(pcr[0]), np.float32(pcr[1]), np.float32(1.0) / np.float32(stride)


def anchor_mask(points, point_cloud_range, grid_size, feature_shape):
    """points [Np, ld] fp32 CUDA (column 1 = x, column 2 = y; all scenes), feature_shape = the shape of the BEV feature
    map (..., H, W) -> bool [H, W] on the points' device, equal to get_anchor_mask's result."""
    ops._require_cuda(points)
    if points.dtype != torch.float32 or points.dim() != 2:
        raise ValueError('anchor_mask: points must be a 2-D fp32 tensor')
    if points.stride(1) != 1:
        points = points.contiguous()
    H, W = int(feature_shape[-2]), int(feature_shape[-1])
    min_x, min_y, inv_stride = mask_params(point_cloud_range, grid_size)
    coarse = torch.zeros((H // 10) * (W // 10), dtype=torch.uint8, device=points.device)
    mask = torch.empty((H, W), dtype=torch.bool, device=points.device)
    check(_lib.load().vc_anchor_mask(points.data_ptr(), points.shape[0], points.stride(0), float(min_x), float(min_y),
                                     float(inv_stride), H, W, coarse.data_ptr(), mask.data_ptr(), ops._stream()),
          'vc_anchor_mask')
    return mask


def ordered_anchors(all_anchors):
    """The reference's output order (axis_aligned_target_assigner.py:121-135): each anchor set viewed as
    (shape[0], shape[1], -1, 7), concatenated along the per-location axis -> (anchors [N, 7] fp32, set index [N] int32)."""
    L = int(all_anchors[0].shape[0]) * int(all_anchors[0].shape[1])
    for a in all_anchors:
        if tuple(a.shape[:2]) != tuple(all_anchors[0].shape[:2]) or a.shape[-1] != 7:
            raise ValueError('anchor sets must share the first two dimensions and have 7 values per anchor')
    per = tuple(a.numel() // (7 * L) if L else 0 for a in all_anchors)
    dev = all_anchors[0].device
    anchors = torch.cat([a.reshape(L, -1, 7) for a in all_anchors], 1).reshape(-1, 7).float().contiguous()
    sid = torch.cat([torch.full((L, n), s, dtype=torch.int32, device=dev) for s, n in enumerate(per)], 1).reshape(-1)
    return anchors, sid


def name_sets(class_names, anchor_class_names):
    """bit s of entry k: anchor set s's class name is class_names[k]"""
    return [sum(1 << s for s, n in enumerate(anchor_class_names) if n == c) for c in class_names]


def assign_targets_batched(anchors, anchor_set, gt_boxes_with_classes, name_sets, matched_thresholds,
                           unmatched_thresholds, out):
    """anchors [N, 7] fp32 and anchor_set [N] int32 (ordered_anchors), gt_boxes_with_classes [B, M, C >= 8] fp32 (class
    last), name_sets (see name_sets()), per-set thresholds (host floats), out = (labels [B, N] int32, targets [B, N, 7],
    reg_weights [B, N], gt_ious [B, N] fp32), all CUDA -> out, every element written.  No host read: capturable."""
    ops._require_cuda(anchors, anchor_set, gt_boxes_with_classes, *out)
    labels, targets, reg_weights, gt_ious = out
    B, M, C = gt_boxes_with_classes.shape
    N = anchors.shape[0]
    S = len(matched_thresholds)
    assert anchors.dtype == torch.float32 and anchors.is_contiguous() and anchor_set.dtype == torch.int32
    assert labels.dtype == torch.int32 and labels.shape == (B, N) and targets.shape == (B, N, 7)
    assert reg_weights.shape == (B, N) and gt_ious.shape == (B, N) and all(t.is_contiguous() for t in out)
    gt = gt_boxes_with_classes
    if gt.dtype != torch.float32 or not gt.is_contiguous():
        gt = gt.float().contiguous()
    lib = _lib.load()
    nbytes = lib.vc_anchor_targets_ws_bytes(B, S, M)
    ws = torch.empty((max(1, nbytes),), dtype=torch.uint8, device=anchors.device)
    check(lib.vc_anchor_targets(anchors.data_ptr(), anchor_set.data_ptr(), N, S, host_f32(matched_thresholds),
                                host_f32(unmatched_thresholds), gt.data_ptr(), B, M, C, host_i32(name_sets),
                                len(name_sets), labels.data_ptr(), targets.data_ptr(), reg_weights.data_ptr(),
                                gt_ious.data_ptr(), ws.data_ptr(), nbytes, ops._stream()), 'vc_anchor_targets')
    return out


class AxisAlignedTargetAssigner(object):
    """`AxisAlignedTargetAssigner` (axis_aligned_target_assigner.py:9-243): same constructor, attributes and
    `assign_targets` result (keys, shapes, dtypes, values), computed by one batched kernel pair."""

    def __init__(self, model_cfg, class_names, box_coder, grid_size, point_cloud_range, match_height=False):
        super().__init__()
        anchor_generator_cfg = model_cfg.ANCHOR_GENERATOR_CONFIG
        anchor_target_cfg = model_cfg.TARGET_ASSIGNER_CONFIG
        self.grid_size = grid_size
        self.point_cloud_range = point_cloud_range
        self.voxel_size = (point_cloud_range[3] - point_cloud_range[0]) / grid_size[0]
        self.feature_map_stride = [config['feature_map_stride'] for config in anchor_generator_cfg]
        self.box_coder = box_coder
        self.match_height = match_height
        self.class_names = np.array(class_names)
        self.anchor_class_names = [config['class_name'] for config in anchor_generator_cfg]
        self.pos_fraction = anchor_target_cfg.POS_FRACTION if anchor_target_cfg.POS_FRACTION >= 0 else None
        self.sample_size = anchor_target_cfg.SAMPLE_SIZE
        self.norm_by_num_examples = anchor_target_cfg.NORM_BY_NUM_EXAMPLES
        self.matched_thresholds = {}
        self.unmatched_thresholds = {}
        for config in anchor_generator_cfg:
            self.matched_thresholds[config['class_name']] = config['matched_threshold']
            self.unmatched_thresholds[config['class_name']] = config['unmatched_threshold']
        self.use_multihead = model_cfg.get('USE_MULTIHEAD', False)
        self.seperate_multihead = model_cfg.get('SEPERATE_MULTIHEAD', False)
        for bad, what in ((self.use_multihead, 'USE_MULTIHEAD'), (match_height, 'MATCH_HEIGHT: True'),
                          (self.pos_fraction is not None, 'POS_FRACTION >= 0 (random subsampling)'),
                          (self.norm_by_num_examples, 'NORM_BY_NUM_EXAMPLES: True'),
                          (getattr(box_coder, 'code_size', None) != 7, 'a box coder with code_size != 7'),
                          (len(self.anchor_class_names) > MAX_SETS, f'more than {MAX_SETS} anchor sets'),
                          (len(class_names) > MAX_NAMES, f'more than {MAX_NAMES} class names')):
            if bad:
                raise ValueError(f'{what}: not supported by the fused target assignment; use {_REF}')
        self._name_sets = name_sets(list(class_names), self.anchor_class_names)
        self._matched = [self.matched_thresholds[n] for n in self.anchor_class_names]
        self._unmatched = [self.unmatched_thresholds[n] for n in self.anchor_class_names]

    def assign_targets(self, all_anchors, gt_boxes_with_classes):
        """all_anchors: [(d0, d1, ..., 7), ...] per anchor set, gt_boxes_with_classes (B, M, 8) -> dict of fresh tensors
        box_cls_labels int32 [B, N], box_reg_targets [B, N, 7], reg_weights / gt_ious fp32 [B, N]"""
        anchors, sid = ordered_anchors(all_anchors)
        B, N = gt_boxes_with_classes.shape[0], anchors.shape[0]
        dev = anchors.device
        out = (torch.empty((B, N), dtype=torch.int32, device=dev), torch.empty((B, N, 7), dtype=torch.float32, device=dev),
               torch.empty((B, N), dtype=torch.float32, device=dev), torch.empty((B, N), dtype=torch.float32, device=dev))
        assign_targets_batched(anchors, sid, gt_boxes_with_classes, self._name_sets, self._matched, self._unmatched, out)
        return {'box_cls_labels': out[0], 'box_reg_targets': out[1], 'reg_weights': out[2], 'gt_ious': out[3]}


def get_anchor_mask(self, data_dict, shape):
    """AnchorHeadSingle.get_anchor_mask on the device (bound by reference_env.install(use_fused_rpn_targets=True))"""
    return anchor_mask(data_dict['points'], self.range, self.grid_size, shape)
