"""RoI target sampling of the two-stage head (TEDMHead of VirConv-L / -T / -S) on the sm_90a kernels of
csrc/roi_targets.cu, which states the rules.

  * `ProposalTargetLayer` = the reference class (roi_heads/target_assigner/proposal_target_layer.py), same constructor
                            and `forward` result dict, all scenes in one batched call;
  * `assign_targets`      = RoIHeadTemplate.assign_targets (roi_head_template.py:121-159) as a drop-in method: with a
                            fused layer the sampling and the canonical transform are one call;
  * `roi_targets_batched` = the same into caller-owned buffers with explicit uniforms, for CUDA-graph capture;
  * `check_status`        = the one host read: raises the reference's error for a scene with neither foreground nor
                            background RoIs.

The reference draws its samples on the host (np.random.permutation / rand / randint, torch.randint).  Here the draws
come from uniforms made by `torch.rand` on the current CUDA generator and mapped to the same laws (rule 4 of the .cu
file), so nothing reads the device on the host.  Supported: SAMPLE_ROI_BY_EACH_CLASS True, CLS_SCORE_TYPE roi_iou_x —
what the VirConv YAMLs use; anything else is rejected at construction: use the reference class for it."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from . import _lib, ops
from ._lib import check, host_f64

MAX_ROIS = 4096     # VC_ROI_TARGETS_MAX_ROIS: RoIs per scene
MAX_GT = 512        # VC_ROI_TARGETS_MAX_GT: GT rows per scene (padded count)
MAX_LDG = 16        # VC_ROI_TARGETS_MAX_LDG: GT columns
MAX_CLASSES = 16    # VC_ROI_TARGETS_MAX_CLASSES: threshold entries
_REF = 'pcdet.models.roi_heads.target_assigner.proposal_target_layer.ProposalTargetLayer (the reference class)'
OUT_KEYS = ('rois', 'gt_of_rois_src', 'gt_of_rois', 'gt_iou_of_rois', 'roi_scores', 'roi_labels', 'reg_valid_mask',
            'rcnn_cls_labels', 'status')


class SamplerConfig:
    """The numbers of a roi_sampler_cfg (TARGET_CONFIG.STAGE*) the kernel takes, validated."""

    def __init__(self, cfg):
        get = cfg.get if hasattr(cfg, 'get') else (lambda k, d=None: getattr(cfg, k, d))
        if get('CLS_SCORE_TYPE') != 'roi_iou_x':
            raise ValueError(f"CLS_SCORE_TYPE {get('CLS_SCORE_TYPE')!r}: only 'roi_iou_x' is supported by the fused "
                             f'RoI target sampling; use {_REF}')
        if not get('SAMPLE_ROI_BY_EACH_CLASS', False):
            raise ValueError(f'SAMPLE_ROI_BY_EACH_CLASS False: not supported by the fused RoI target sampling; use {_REF}')
        self.reg_fg = [float(v) for v in cfg.REG_FG_THRESH]
        self.cls_fg = [float(v) for v in cfg.CLS_FG_THRESH]
        self.cls_bg = [float(v) for v in cfg.CLS_BG_THRESH]
        n = len(self.reg_fg)
        if n > MAX_CLASSES:
            raise ValueError(f'{n} classes: more than the {MAX_CLASSES} the fused RoI target sampling supports; use {_REF}')
        if n == 0 or len(self.cls_fg) != n or len(self.cls_bg) != n:
            raise ValueError(f'REG_FG_THRESH, CLS_FG_THRESH and CLS_BG_THRESH must have one entry per class; use {_REF}')
        self.n_cls = n
        self.lo = float(cfg.CLS_BG_THRESH_LO)
        self.R = int(cfg.ROI_PER_IMAGE)
        self.F = int(np.round(cfg.FG_RATIO * cfg.ROI_PER_IMAGE))
        if not 0 <= self.F <= self.R:
            raise ValueError(f'FG_RATIO {cfg.FG_RATIO} outside [0, 1]; use {_REF}')
        self.hard_bg_ratio = float(cfg.HARD_BG_RATIO)
        self.hard_sampling = bool(get('ENABLE_HARD_SAMPLING', False))
        self.hs_thresh = [float(v) for v in cfg.HARD_SAMPLING_THRESH] if self.hard_sampling else [0.0] * n
        self.hs_ratio = [float(v) for v in cfg.HARD_SAMPLING_RATIO] if self.hard_sampling else [1.0] * n
        if len(self.hs_thresh) < n or len(self.hs_ratio) < n or any(int(1 / r) < 1 for r in self.hs_ratio):
            raise ValueError(f'HARD_SAMPLING_THRESH / HARD_SAMPLING_RATIO need one entry per class, ratios in (0, 1]; '
                             f'use {_REF}')


def draw_uniforms(B, M, R, n_cls, device):
    """(u_fg [B, max(M, R)], u_bg [B, R], u_hs [n_cls]) from torch.rand on the current CUDA generator"""
    return (torch.rand((B, max(M, R)), device=device), torch.rand((B, R), device=device),
            torch.rand((n_cls,), device=device))


def empty_outputs(B, R, roi_code_size, gt_code_size, device):
    """caller-owned output buffers for roi_targets_batched, keyed as OUT_KEYS"""
    f = dict(dtype=torch.float32, device=device)
    return {'rois': torch.empty((B, R, roi_code_size), **f), 'gt_of_rois_src': torch.empty((B, R, gt_code_size), **f),
            'gt_of_rois': torch.empty((B, R, gt_code_size), **f), 'gt_iou_of_rois': torch.empty((B, R), **f),
            'roi_scores': torch.empty((B, R), **f), 'roi_labels': torch.empty((B, R), dtype=torch.int64, device=device),
            'reg_valid_mask': torch.empty((B, R), dtype=torch.int64, device=device),
            'rcnn_cls_labels': torch.empty((B, R), **f), 'status': torch.empty((1,), dtype=torch.int32, device=device)}


def roi_targets_batched(cfg, rois, roi_scores, roi_labels, gt_boxes, uniforms, out):
    """cfg: a SamplerConfig; rois [B, M, >= 7], roi_scores [B, M] fp32, roi_labels [B, M] int64, gt_boxes [B, G, >= 8]
    (class last), uniforms = (u_fg [B, >= max(M, R)], u_bg [B, R], u_hs [n_cls]) in [0, 1), out = empty_outputs(...),
    all CUDA -> out, every element written (gt_of_rois canonical, gt_of_rois_src as gathered; status [1] = number of
    scenes with neither foreground nor background).  No host read: capturable."""
    u_fg, u_bg, u_hs = uniforms
    ops._require_cuda(rois, roi_scores, roi_labels, gt_boxes, u_fg, u_bg, u_hs, *out.values())
    B, M, ldr = rois.shape
    G, ldg = gt_boxes.shape[1], gt_boxes.shape[2]
    R = cfg.R
    if rois.dtype != torch.float32 or gt_boxes.dtype != torch.float32 or roi_scores.dtype != torch.float32:
        raise ValueError('roi_targets_batched: rois, roi_scores and gt_boxes must be fp32')
    assert roi_labels.dtype == torch.int64 and roi_labels.shape == (B, M) and roi_scores.shape == (B, M)
    assert gt_boxes.shape[0] == B and u_fg.shape[0] == B and u_fg.shape[1] >= max(M, R) and u_bg.shape == (B, R)
    assert u_hs.numel() >= cfg.n_cls and all(u.dtype == torch.float32 for u in uniforms)
    assert out['rois'].shape == (B, R, ldr) and out['gt_of_rois'].shape == (B, R, ldg)
    assert all(t.is_contiguous() for t in out.values())
    rois, roi_scores, roi_labels, gt_boxes = (t.contiguous() for t in (rois, roi_scores, roi_labels, gt_boxes))
    u_fg, u_bg, u_hs = (u.contiguous() for u in uniforms)
    lib = _lib.load()
    nbytes = lib.vc_roi_targets_ws_bytes(B, M, G)
    ws = torch.empty((max(1, nbytes),), dtype=torch.uint8, device=rois.device)
    o = out
    check(lib.vc_roi_targets(rois.data_ptr(), roi_scores.data_ptr(), roi_labels.data_ptr(), B, M, ldr, gt_boxes.data_ptr(),
                             G, ldg, cfg.n_cls, host_f64(cfg.reg_fg), host_f64(cfg.cls_fg), host_f64(cfg.cls_bg), cfg.lo,
                             host_f64(cfg.hs_thresh), host_f64(cfg.hs_ratio), int(cfg.hard_sampling), R, cfg.F,
                             cfg.hard_bg_ratio, u_fg.data_ptr(), u_fg.stride(0), u_bg.data_ptr(), u_hs.data_ptr(),
                             o['rois'].data_ptr(), o['gt_of_rois_src'].data_ptr(), o['gt_of_rois'].data_ptr(),
                             o['gt_iou_of_rois'].data_ptr(), o['roi_scores'].data_ptr(), o['roi_labels'].data_ptr(),
                             o['reg_valid_mask'].data_ptr(), o['rcnn_cls_labels'].data_ptr(), o['status'].data_ptr(),
                             ws.data_ptr(), nbytes, ops._stream()), 'vc_roi_targets')
    return out


def check_status(status):
    """The one host read: raises NotImplementedError, as ProposalTargetLayer.subsample_rois does, when a scene had
    neither foreground nor background RoIs (its output rows are zero)."""
    n = int(status.reshape(-1)[0].item())
    if n:
        raise NotImplementedError(f'ERROR: FG=0, BG=0 in {n} scene(s): no RoI to sample (ProposalTargetLayer)')


class ProposalTargetLayer(nn.Module):
    """`ProposalTargetLayer` (proposal_target_layer.py:7-389): same constructor and `forward(batch_dict, ind)` result
    (keys, shapes, dtypes; the values the reference gives with the same draws), one batched kernel pair, no host read.
    A scene with neither foreground nor background RoIs gets zero rows instead of the reference's exception; the status
    word of the last call (`self.last_status`) tells, through check_status."""

    def __init__(self, roi_sampler_cfg):
        super().__init__()
        self.roi_sampler_cfg = roi_sampler_cfg
        self._cfg = SamplerConfig(roi_sampler_cfg)
        self.last_status = None

    def sample(self, batch_dict, ind=''):
        """all outputs of roi_targets_batched (gt_of_rois canonical, gt_of_rois_src as gathered), fresh uniforms"""
        rois, gt = batch_dict['rois'], batch_dict['gt_boxes' + ind]
        B, M = rois.shape[0], rois.shape[1]
        out = empty_outputs(B, self._cfg.R, rois.shape[-1], gt.shape[-1], rois.device)
        uniforms = draw_uniforms(B, M, self._cfg.R, self._cfg.n_cls, rois.device)
        roi_targets_batched(self._cfg, rois.float(), batch_dict['roi_scores'].float(), batch_dict['roi_labels'].long(),
                            gt.float(), uniforms, out)
        self.last_status = out['status']
        return out

    def forward(self, batch_dict, ind=''):
        out = self.sample(batch_dict, ind)
        return {'rois': out['rois'], 'gt_of_rois': out['gt_of_rois_src'], 'gt_iou_of_rois': out['gt_iou_of_rois'],
                'roi_scores': out['roi_scores'], 'roi_labels': out['roi_labels'],
                'reg_valid_mask': out['reg_valid_mask'], 'rcnn_cls_labels': out['rcnn_cls_labels']}


_reference_assign_targets = None    # RoIHeadTemplate.assign_targets as the reference defines it (set by reference_env)


def assign_targets(self, batch_dict, rot_num_id, enable_dif=False):
    """RoIHeadTemplate.assign_targets (bound by reference_env.install(use_fused_roi_targets=True)).  With a fused layer:
    one call that samples and applies the canonical transform; with the reference layer: the reference method."""
    layer = self.proposal_target_layers[rot_num_id]
    s_str = '' if rot_num_id == 0 else str(rot_num_id)
    ind = s_str if enable_dif else ''
    if isinstance(layer, ProposalTargetLayer):
        with torch.no_grad():
            out = layer.sample(batch_dict, ind)
        return {'rois': out['rois'], 'gt_of_rois': out['gt_of_rois'], 'gt_iou_of_rois': out['gt_iou_of_rois'],
                'roi_scores': out['roi_scores'], 'roi_labels': out['roi_labels'],
                'reg_valid_mask': out['reg_valid_mask'], 'rcnn_cls_labels': out['rcnn_cls_labels'],
                'gt_of_rois_src': out['gt_of_rois_src']}
    if _reference_assign_targets is None:
        raise RuntimeError('assign_targets: a reference ProposalTargetLayer needs the reference method, which '
                           'reference_env.install(use_fused_roi_targets=True) records before binding this one')
    return _reference_assign_targets(self, batch_dict, rot_num_id, enable_dif)
