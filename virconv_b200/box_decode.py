"""Box decoding of the RPN and RCNN heads and TEDMHead's cascade stage transforms on the sm_90a kernels of
csrc/box_decode.cu, which states the rules.

  * `anchor_decode`  = ResidualCoder.decode_torch + the direction-classifier heading of
                       AnchorHeadTemplate.generate_predicted_boxes (anchor_head_template.py:335-382), all scenes in one
                       launch, as a torch.autograd.Function differentiable with respect to box_preds;
  * `roi_decode`     = the decode, rotation and translation of RoIHeadTemplate.generate_predicted_boxes
                       (roi_head_template.py:294-324), as a torch.autograd.Function differentiable with respect to
                       box_preds;
  * `box_xtrans`     = X_TRANS.backward_with_param of one stage then forward_with_param of another (X_transform.py:49-154)
                       on the boxes of all scenes, the parameters read on the device;
  * `anchor_generate_predicted_boxes`, `roi_generate_predicted_boxes`, `roi_x_trans`, `roi_score_trans`,
    `pred_x_trans` = the drop-in methods (bound by reference_env.install(use_fused_box_decode=True)).

The reference decodes in a few dozen small elementwise kernels and rotates through a batched 3 x 3 matmul; its stage
transforms loop over the scenes in Python and read the device in `world_flip` (`if enable` on a CUDA scalar,
augmentor_utils.py:28) once per transform and scene.  Here each call is one launch and nothing reads the device, so a
stage loop can be captured in a CUDA graph.

Fallbacks to the reference method: RoIs that require a gradient in roi_generate_predicted_boxes (the reference
differentiates them through the rotation; VirConv's RoIs come from assign_targets under no_grad), and boxes that require a
gradient in the three stage transforms (in training the previous stage's predictions, which carry rcnn_reg's graph).
Configurations VirConv does not use raise ValueError naming the reference method."""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, ops
from ._lib import check

XTRANS_ORDER = ('world_rotation', 'world_flip', 'world_scaling')   # X_TRANS's default AUG_CONFIG_LIST, TEDMHead's
_AHT = 'pcdet.models.dense_heads.anchor_head_template.AnchorHeadTemplate.generate_predicted_boxes'
_RHT = 'pcdet.models.roi_heads.roi_head_template.RoIHeadTemplate.generate_predicted_boxes'
_TED = 'pcdet.models.roi_heads.ted_head.TEDMHead.'

_reference_anchor_generate_predicted_boxes = None   # the reference methods (set by reference_env)
_reference_roi_generate_predicted_boxes = None
_reference_roi_x_trans = None
_reference_roi_score_trans = None
_reference_pred_x_trans = None


def _f32(v):
    """v as the float32 value torch's wrapped-scalar rule gives a float32 tensor op"""
    return float(np.float32(v))


def _require_f32(what, ref, *tensors):
    for t in tensors:
        if t is not None and t.dtype != torch.float32:
            raise ValueError(f'{what}: float32 tensors only (got {t.dtype}); use {ref}')


class _AnchorDecode(torch.autograd.Function):
    @staticmethod
    def forward(ctx, box, dir_cls, anchors, dir_offset, dir_limit_offset, period):
        box_c, anc_c = box.contiguous(), anchors.contiguous()
        dir_c = dir_cls.contiguous() if dir_cls is not None else None
        B, A = box_c.shape[0], box_c.shape[1]
        NB = dir_c.shape[-1] if dir_c is not None else 0
        out = torch.empty((B, A, 7), dtype=torch.float32, device=box.device)
        check(_lib.load().vc_anchor_decode(box_c.data_ptr(), ops._p(dir_c), anc_c.data_ptr(), B, A, NB,
                                           _f32(dir_offset), _f32(dir_limit_offset), _f32(period), out.data_ptr(),
                                           ops._stream()), 'vc_anchor_decode')
        ctx.save_for_backward(box_c, anc_c)
        ctx.with_dir = dir_c is not None
        return out

    @staticmethod
    def backward(ctx, grad_out):
        if not ctx.needs_input_grad[0]:
            return None, None, None, None, None, None
        box, anchors = ctx.saved_tensors
        g = grad_out.contiguous()
        dbox = torch.empty_like(box)
        check(_lib.load().vc_anchor_decode_bwd(g.data_ptr(), box.data_ptr(), anchors.data_ptr(), box.shape[0],
                                               box.shape[1], int(ctx.with_dir), dbox.data_ptr(), ops._stream()),
              'vc_anchor_decode_bwd')
        return dbox, None, None, None, None, None


def anchor_decode(box_preds, anchors, dir_cls_preds=None, dir_offset=0.0, dir_limit_offset=0.0, period=np.pi):
    """box_preds [B, A, 7] residuals, anchors [A, 7] shared by the scenes, dir_cls_preds [B, A, NB] or None, CUDA fp32 ->
    boxes [B, A, 7]: ResidualCoder.decode_torch, then with dir_cls_preds the heading limit_period(h - dir_offset,
    dir_limit_offset, period) + dir_offset + period * argmax.  Differentiable with respect to box_preds only.  One
    launch; no host read."""
    ops._require_cuda(box_preds, anchors, dir_cls_preds)
    _require_f32('anchor_decode', _AHT, box_preds, anchors, dir_cls_preds)
    if box_preds.dim() != 3 or box_preds.shape[2] != 7:
        raise ValueError(f'anchor_decode: box_preds {tuple(box_preds.shape)} is not [B, A, 7]; use {_AHT}')
    B, A = box_preds.shape[:2]
    if tuple(anchors.shape) != (A, 7):
        raise ValueError(f'anchor_decode: anchors {tuple(anchors.shape)} is not [{A}, 7]; use {_AHT}')
    if dir_cls_preds is not None and (dir_cls_preds.dim() != 3 or tuple(dir_cls_preds.shape[:2]) != (B, A)
                                      or dir_cls_preds.shape[2] < 1):
        raise ValueError(f'anchor_decode: dir_cls_preds {tuple(dir_cls_preds.shape)} is not [{B}, {A}, NB]; use {_AHT}')
    return _AnchorDecode.apply(box_preds, dir_cls_preds, anchors, dir_offset, dir_limit_offset, period)


class _RoiDecode(torch.autograd.Function):
    @staticmethod
    def forward(ctx, box, rois):
        box_c, rois_c = box.contiguous(), rois.contiguous()
        B, N, ld = rois_c.shape
        out = torch.empty((B, N, 7), dtype=torch.float32, device=box.device)
        check(_lib.load().vc_roi_decode(box_c.data_ptr(), rois_c.data_ptr(), B, N, ld, out.data_ptr(), ops._stream()),
              'vc_roi_decode')
        ctx.save_for_backward(box_c, rois_c)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        if not ctx.needs_input_grad[0]:
            return None, None
        box, rois = ctx.saved_tensors
        B, N, ld = rois.shape
        g = grad_out.contiguous()
        dbox = torch.empty_like(box)
        check(_lib.load().vc_roi_decode_bwd(g.data_ptr(), box.data_ptr(), rois.data_ptr(), B, N, ld, dbox.data_ptr(),
                                            ops._stream()), 'vc_roi_decode_bwd')
        return dbox, None


def roi_decode(box_preds, rois):
    """box_preds [B * N, 7] residuals, rois [B, N, >= 7], CUDA fp32 -> boxes [B, N, 7]: decoded against the RoI at the
    origin, rotated by its heading and moved to its centre.  Differentiable with respect to box_preds only (RoIs that
    require a gradient raise: the drop-in method sends them to the reference).  One launch; no host read."""
    ops._require_cuda(box_preds, rois)
    _require_f32('roi_decode', _RHT, box_preds, rois)
    if rois.dim() != 3 or rois.shape[2] < 7:
        raise ValueError(f'roi_decode: rois {tuple(rois.shape)} is not [B, N, >= 7]; use {_RHT}')
    B, N = rois.shape[:2]
    if tuple(box_preds.shape) != (B * N, 7):
        raise ValueError(f'roi_decode: box_preds {tuple(box_preds.shape)} is not [{B * N}, 7]; use {_RHT}')
    if rois.requires_grad:
        raise ValueError(f'roi_decode: rois that require a gradient; use {_RHT}')
    return _RoiDecode.apply(box_preds, rois)


def _stage(i, R):
    """a stage of transform_param[b]: Python's index rule (-1 is the last stage); None -> no transform (-1)"""
    if i is None:
        return -1
    i = int(i)
    if not -R <= i < R:
        raise IndexError(f'box_xtrans: stage {i} of {R}')
    return i + R if i < 0 else i


def box_xtrans(boxes, transform_param, from_stage, to_stage):
    """boxes [B, N, >= 7], transform_param [B', R, 3] (rotation, flip, scale; B' >= B), CUDA fp32 -> [B, N, same]: each
    scene's boxes taken back through X_TRANS.backward_with_param of stage `from_stage`, then through
    forward_with_param of stage `to_stage` (either None: skipped; negative stages index from the end, as Python's).
    Columns beyond 7 are copied.  One launch; the parameters are read on the device."""
    ops._require_cuda(boxes, transform_param)
    _require_f32('box_xtrans', _TED + 'roi_x_trans', boxes, transform_param)
    if boxes.dim() != 3 or boxes.shape[2] < 7:
        raise ValueError(f'box_xtrans: boxes {tuple(boxes.shape)} is not [B, N, >= 7]; use {_TED}roi_x_trans')
    if transform_param.dim() != 3 or transform_param.shape[2] != 3 or transform_param.shape[0] < boxes.shape[0]:
        raise ValueError(f'box_xtrans: transform_param {tuple(transform_param.shape)} is not [{boxes.shape[0]}, R, 3] '
                         f'(rotation, flip, scale); use {_TED}roi_x_trans')
    R = transform_param.shape[1]
    f, t = _stage(from_stage, R), _stage(to_stage, R)
    b, p = boxes.contiguous(), transform_param.contiguous()
    B, N, ld = b.shape
    out = torch.empty_like(b)
    check(_lib.load().vc_box_xtrans(b.data_ptr(), p.data_ptr(), B, N, ld, R, f, t, out.data_ptr(), ops._stream()),
          'vc_box_xtrans')
    return out


# ---- drop-in methods -------------------------------------------------------------------------------------------------
def _residual_coder(coder, ref):
    name = type(coder).__name__
    if name == 'PreviousResidualDecoder':
        raise ValueError(f'generate_predicted_boxes: PreviousResidualDecoder is not supported by the fused decode; use {ref}')
    if name != 'ResidualCoder' or getattr(coder, 'encode_angle_by_sincos', False) or coder.code_size != 7:
        raise ValueError(f'generate_predicted_boxes: box coder {name} with code size {getattr(coder, "code_size", None)}; '
                         f'the fused decode takes ResidualCoder with 7 codes; use {ref}')


def anchor_generate_predicted_boxes(self, batch_size, cls_preds, box_preds, dir_cls_preds=None):
    """AnchorHeadTemplate.generate_predicted_boxes (bound by reference_env.install(use_fused_box_decode=True)):
    -> (batch_cls_preds [B, A, C], the reference's view of cls_preds; batch_box_preds [B, A, 7], one launch)."""
    _residual_coder(self.box_coder, _AHT)
    anchors = self.anchors
    if isinstance(anchors, list):
        if getattr(self, 'use_multihead', False):
            raise ValueError(f'generate_predicted_boxes: multihead anchors; use {_AHT}')
        anchors = anchors[0] if len(anchors) == 1 else torch.cat(anchors, dim=-3)
    if any(isinstance(x, list) for x in (cls_preds, box_preds, dir_cls_preds)):
        raise ValueError(f'generate_predicted_boxes: list-form predictions; use {_AHT}')
    if anchors.shape[-1] != 7:
        raise ValueError(f'generate_predicted_boxes: anchors with {anchors.shape[-1]} columns; use {_AHT}')
    _require_f32('generate_predicted_boxes', _AHT, box_preds, anchors, dir_cls_preds)
    anchors = anchors.reshape(-1, 7)
    num_anchors = anchors.shape[0]
    batch_cls_preds = cls_preds.view(batch_size, num_anchors, -1).float()
    box = box_preds.view(batch_size, num_anchors, -1)
    if dir_cls_preds is None:
        return batch_cls_preds, anchor_decode(box, anchors)
    cfg = self.model_cfg
    dirs = dir_cls_preds.view(batch_size, num_anchors, -1)
    return batch_cls_preds, anchor_decode(box, anchors, dirs, cfg.DIR_OFFSET, cfg.DIR_LIMIT_OFFSET,
                                          2 * np.pi / cfg.NUM_DIR_BINS)


def roi_generate_predicted_boxes(self, batch_size, rois, cls_preds, box_preds):
    """RoIHeadTemplate.generate_predicted_boxes (bound by reference_env.install(use_fused_box_decode=True)):
    -> (batch_cls_preds [B, N, C], the reference's view of cls_preds; batch_box_preds [B, N, 7], one launch).  RoIs that
    require a gradient go to the reference method."""
    if rois.requires_grad:
        if _reference_roi_generate_predicted_boxes is None:
            raise RuntimeError('generate_predicted_boxes: RoIs that require a gradient need the reference method, which '
                               'reference_env.install(use_fused_box_decode=True) records before binding this one')
        return _reference_roi_generate_predicted_boxes(self, batch_size, rois, cls_preds, box_preds)
    _residual_coder(self.box_coder, _RHT)
    batch_cls_preds = cls_preds.view(batch_size, -1, cls_preds.shape[-1])
    return batch_cls_preds, roi_decode(box_preds.view(-1, 7), rois)


def _xtrans_method(name, reference, self, boxes, rot_num_id, transform_param, stages):
    if boxes.requires_grad:
        if reference is None:
            raise RuntimeError(f'{name}: boxes that require a gradient need the reference method, which '
                               f'reference_env.install(use_fused_box_decode=True) records before binding this one')
        return reference(self, boxes, rot_num_id, transform_param)
    cfgs = self.x_trans_train.aug_config_list
    names = tuple(c['NAME'] for c in cfgs)
    if names != XTRANS_ORDER:
        raise ValueError(f'{name}: X_TRANS augmentors {names}; the fused transform takes {XTRANS_ORDER}; '
                         f'use {_TED}{name}')
    R = transform_param.shape[1]
    while rot_num_id >= R:
        rot_num_id -= 1
    return box_xtrans(boxes, transform_param, *stages(rot_num_id))


def roi_x_trans(self, rois, rot_num_id, transform_param):
    """TEDMHead.roi_x_trans (bound by reference_env.install(use_fused_box_decode=True)): stage rot_num_id - 1's
    backward transform, then stage rot_num_id's forward transform, all scenes in one launch."""
    return _xtrans_method('roi_x_trans', _reference_roi_x_trans, self, rois, rot_num_id, transform_param,
                          lambda i: (i - 1, i))


def roi_score_trans(self, rois, rot_num_id, transform_param):
    """TEDMHead.roi_score_trans (bound by reference_env.install(use_fused_box_decode=True)): stage rot_num_id's
    backward transform, then stage 0's forward transform, all scenes in one launch."""
    return _xtrans_method('roi_score_trans', _reference_roi_score_trans, self, rois, rot_num_id, transform_param,
                          lambda i: (i, 0))


def pred_x_trans(self, preds, rot_num_id, transform_param):
    """TEDMHead.pred_x_trans (bound by reference_env.install(use_fused_box_decode=True)): stage rot_num_id's backward
    transform, all scenes in one launch."""
    return _xtrans_method('pred_x_trans', _reference_pred_x_trans, self, preds, rot_num_id, transform_param,
                          lambda i: (i, None))
