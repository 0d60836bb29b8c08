"""Training losses of the detector heads (AnchorHeadSingle and TEDMHead of VirConv-L / -T / -S) with their gradients, on
the sm_90a kernels of csrc/head_losses.cu, which states the rules.

  * `rpn_loss`             = AnchorHeadTemplate.get_loss (anchor_head_template.py:178-333) as a torch.autograd.Function;
  * `rcnn_loss`            = RoIHeadTemplate.get_loss (roi_head_template.py:161-291), every branch in one launch;
  * `anchor_head_get_loss` / `roi_head_get_loss` = the drop-in methods (bound by
                             reference_env.install(use_fused_losses=True)): same `(loss, tb_dict)`, the tb floats from one
                             device-to-host copy.

The forwards write the losses and d loss / d prediction in one call each and read nothing back on the host; the
backwards scale the saved gradients by the incoming gradient.  Both can be captured in a CUDA graph.  Supported: OD_LOSS
off, the reference's WeightedSmoothL1Loss, one head, a 7-value ResidualCoder for the RPN; CLS_LOSS BinaryCrossEntropy and
REG_LOSS smooth-l1 for the RCNN — what the VirConv YAMLs use.  Anything else is rejected at construction: use the
reference method for it."""
from __future__ import annotations

import ctypes

import torch

from . import _lib, ops
from ._lib import check, host_f64
from .anchor_targets import ordered_anchors

MAX_BRANCHES = 18   # VC_RCNN_MAX_BRANCHES: 6 stages x 3 branches, the reference's loop bound
_REF_RPN = 'pcdet.models.dense_heads.anchor_head_template.AnchorHeadTemplate.get_loss (the reference method)'
_REF_RCNN = 'pcdet.models.roi_heads.roi_head_template.RoIHeadTemplate.get_loss (the reference method)'
BRANCH_KEYS = (('targets_dict', 1.0), ('targets_dict_pi', 0.5), ('targets_dict_p', 0.5))


def _get(cfg, key, default=None):
    return cfg.get(key, default) if hasattr(cfg, 'get') else getattr(cfg, key, default)


def _code_weights(weights, ref):
    cw = [float(v) for v in weights['code_weights']]
    if len(cw) != 7:
        raise ValueError(f'{len(cw)} code weights: only a code size of 7 is supported by the fused loss; use {ref}')
    return cw


class RPNLossConfig:
    """The numbers of a DENSE_HEAD config that vc_rpn_loss takes, validated."""

    def __init__(self, model_cfg, num_class):
        lc = model_cfg.LOSS_CONFIG
        tac = _get(model_cfg, 'TARGET_ASSIGNER_CONFIG', {}) or {}
        bcc = _get(tac, 'BOX_CODER_CONFIG', {}) or {}
        reg_type = _get(lc, 'REG_LOSS_TYPE', None)
        for bad, what in ((_get(model_cfg, 'OD_LOSS', False), 'OD_LOSS (odiou)'),
                          (reg_type not in (None, 'WeightedSmoothL1Loss'), f'REG_LOSS_TYPE {reg_type!r}'),
                          (_get(model_cfg, 'USE_MULTIHEAD', False), 'USE_MULTIHEAD'),
                          (_get(bcc, 'encode_angle_by_sincos', False), 'encode_angle_by_sincos'),
                          (_get(tac, 'BOX_CODER', 'ResidualCoder') != 'ResidualCoder', 'a box coder other than ResidualCoder'),
                          (int(_get(bcc, 'code_size', 7)) != 7, 'a code size other than 7')):
            if bad:
                raise ValueError(f'{what}: not supported by the fused RPN loss; use {_REF_RPN}')
        w = lc.LOSS_WEIGHTS
        self.code_weights = _code_weights(w, _REF_RPN)
        self.num_class = int(num_class)
        self.alpha, self.gamma, self.beta = 0.25, 2.0, 1.0 / 9.0     # build_losses (:145-159)
        self.cls_weight = float(w['cls_weight'])
        self.loc_weight = float(w['loc_weight'])
        self.dir_weight = float(w.get('dir_weight', 0.0))
        self.dir_offset = float(_get(model_cfg, 'DIR_OFFSET', 0.0))
        self.num_dir_bins = int(_get(model_cfg, 'NUM_DIR_BINS', 2))


class RCNNLossConfig:
    """The numbers of a ROI_HEAD config that vc_rcnn_loss takes, validated."""

    def __init__(self, model_cfg):
        lc = model_cfg.LOSS_CONFIG
        if lc.CLS_LOSS != 'BinaryCrossEntropy':
            raise ValueError(f'CLS_LOSS {lc.CLS_LOSS!r}: only BinaryCrossEntropy is supported by the fused RCNN loss; '
                             f'use {_REF_RCNN}')
        if lc.REG_LOSS != 'smooth-l1':
            raise ValueError(f'REG_LOSS {lc.REG_LOSS!r}: only smooth-l1 is supported by the fused RCNN loss; use {_REF_RCNN}')
        tc = _get(model_cfg, 'TARGET_CONFIG', {}) or {}
        bcc = _get(tc, 'BOX_CODER_CONFIG', {}) or {}
        if _get(bcc, 'encode_angle_by_sincos', False) or int(_get(bcc, 'code_size', 7)) != 7:
            raise ValueError(f'a box coder other than the 7-value ResidualCoder: not supported by the fused RCNN loss; '
                             f'use {_REF_RCNN}')
        w = lc.LOSS_WEIGHTS
        self.code_weights = _code_weights(w, _REF_RCNN)
        self.beta = 1.0 / 9.0
        self.cls_weight = float(w['rcnn_cls_weight'])
        self.reg_weight = float(w['rcnn_reg_weight'])
        self.corner = bool(_get(lc, 'CORNER_LOSS_REGULARIZATION', False))
        self.corner_weight = float(w['rcnn_corner_weight']) if self.corner else 0.0


def _f32(t, what):
    if t.dtype != torch.float32:
        raise ValueError(f'{what}: expected a float32 tensor, got {t.dtype}')
    return t.contiguous()


class _RPNLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cls_preds, box_preds, dir_cls_preds, labels, reg_targets, anchors, cfg):
        ops._require_cuda(cls_preds, box_preds, dir_cls_preds, labels, reg_targets, anchors)
        B = int(cls_preds.shape[0])
        cls_c, box_c = _f32(cls_preds, 'cls_preds'), _f32(box_preds, 'box_preds')
        N = box_c.numel() // (B * 7)
        if box_c.numel() != B * N * 7 or cls_c.numel() != B * N * cfg.num_class:
            raise ValueError(f'rpn_loss: box_preds {tuple(box_preds.shape)} / cls_preds {tuple(cls_preds.shape)} do not '
                             f'hold 7 / {cfg.num_class} values per anchor')
        labels = labels.reshape(B, N)
        labels = labels if labels.dtype == torch.int32 and labels.is_contiguous() else labels.to(torch.int32).contiguous()
        tgt = _f32(reg_targets, 'box_reg_targets')
        assert tgt.numel() == B * N * 7
        dir_c = None
        if dir_cls_preds is not None:
            dir_c = _f32(dir_cls_preds, 'dir_cls_preds')
            assert dir_c.numel() == B * N * cfg.num_dir_bins and anchors.shape == (N, 7)
        anc = _f32(anchors, 'anchors')
        dev = cls_c.device
        stats = torch.empty(4, dtype=torch.float32, device=dev)
        g_cls, g_box = torch.empty_like(cls_c), torch.empty_like(box_c)
        g_dir = torch.empty_like(dir_c) if dir_c is not None else None
        lib = _lib.load()
        nbytes = lib.vc_rpn_loss_ws_bytes(B, N)
        ws = torch.empty((max(1, nbytes),), dtype=torch.uint8, device=dev)
        check(lib.vc_rpn_loss(cls_c.data_ptr(), box_c.data_ptr(), ops._p(dir_c), labels.data_ptr(), tgt.data_ptr(),
                              anc.data_ptr(), B, N, cfg.num_class, cfg.num_dir_bins, cfg.alpha, cfg.gamma, cfg.beta,
                              host_f64(cfg.code_weights), cfg.cls_weight, cfg.loc_weight, cfg.dir_weight, cfg.dir_offset,
                              stats.data_ptr(), g_cls.data_ptr(), g_box.data_ptr(), ops._p(g_dir), ws.data_ptr(), nbytes,
                              ops._stream()), 'vc_rpn_loss')
        ctx.save_for_backward(g_cls, g_box, g_dir)
        ctx.shapes = (cls_preds.shape, box_preds.shape, None if dir_cls_preds is None else dir_cls_preds.shape)
        ctx.mark_non_differentiable(stats)
        return stats[3].clone(), stats

    @staticmethod
    def backward(ctx, grad_loss, grad_stats):
        g_cls, g_box, g_dir = ctx.saved_tensors
        s_cls, s_box, s_dir = ctx.shapes
        return ((g_cls * grad_loss).view(s_cls), (g_box * grad_loss).view(s_box),
                None if g_dir is None else (g_dir * grad_loss).view(s_dir), None, None, None, None)


def rpn_loss(cls_preds, box_preds, dir_cls_preds, box_cls_labels, box_reg_targets, anchors, cfg):
    """cls_preds [B, ..., n_cls per anchor], box_preds [B, ..., 7 per anchor], dir_cls_preds [B, ..., bins per anchor]
    or None (as forward_ret_dict holds them), box_cls_labels [B, N], box_reg_targets [B, N, 7], anchors [N, 7] (the
    reference's torch.cat(self.anchors, dim=-3).view(-1, 7); ordered_anchors), cfg = RPNLossConfig, all CUDA ->
    (loss: 0-d tensor = rpn_loss, stats: detached fp32 [4] = rpn_loss_cls, rpn_loss_loc, rpn_loss_dir, rpn_loss).
    No host read: capturable."""
    return _RPNLoss.apply(cls_preds, box_preds, dir_cls_preds, box_cls_labels, box_reg_targets, anchors, cfg)


class _Branch(ctypes.Structure):
    _fields_ = [('rcnn_cls', ctypes.c_void_p), ('rcnn_reg', ctypes.c_void_p), ('rois', ctypes.c_void_p),
                ('gt_of_rois', ctypes.c_void_p), ('gt_of_rois_src', ctypes.c_void_p),
                ('reg_valid_mask', ctypes.c_void_p), ('rcnn_cls_labels', ctypes.c_void_p), ('g_cls', ctypes.c_void_p),
                ('g_reg', ctypes.c_void_p), ('n', ctypes.c_int), ('ldr', ctypes.c_int), ('ldg', ctypes.c_int),
                ('weight', ctypes.c_float)]


class _RCNNLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cfg, weights, targets, *preds):
        K = len(weights)
        dev = preds[0].device
        keep, table, grads = [], (_Branch * K)(), []
        for k in range(K):
            cls, reg = _f32(preds[2 * k], 'rcnn_cls'), _f32(preds[2 * k + 1], 'rcnn_reg')
            t = targets[k]
            rois, gt = _f32(t['rois'], 'rois'), _f32(t['gt_of_rois'], 'gt_of_rois')
            src = _f32(t['gt_of_rois_src'], 'gt_of_rois_src')
            valid = t['reg_valid_mask'].to(torch.int64).contiguous()
            labels = t['rcnn_cls_labels'].to(torch.float32).contiguous()
            n = valid.numel()
            ldr, ldg = rois.shape[-1], gt.shape[-1]
            if ldr != 7 or rois.numel() != n * 7 or gt.numel() != n * ldg or src.shape != gt.shape:
                raise ValueError(f'rcnn_loss: branch {k}: rois {tuple(rois.shape)} (the reference views them as (-1, 7)), '
                                 f'gt_of_rois {tuple(gt.shape)}, gt_of_rois_src {tuple(src.shape)}, {n} rows')
            if cls.numel() != n or reg.numel() != n * 7 or labels.numel() != n:
                raise ValueError(f'rcnn_loss: branch {k}: rcnn_cls {tuple(cls.shape)} / rcnn_reg {tuple(reg.shape)} do '
                                 f'not match {n} RoIs')
            ops._require_cuda(cls, reg, rois, gt, src, valid, labels)
            g_cls, g_reg = torch.empty_like(cls), torch.empty_like(reg)
            table[k] = _Branch(cls.data_ptr(), reg.data_ptr(), rois.data_ptr(), gt.data_ptr(), src.data_ptr(),
                               valid.data_ptr(), labels.data_ptr(), g_cls.data_ptr(), g_reg.data_ptr(), n, ldr, ldg,
                               float(weights[k]))
            keep += [cls, reg, rois, gt, src, valid, labels]
            grads += [g_cls, g_reg]
        stats = torch.empty(K * 4 + 1, dtype=torch.float32, device=dev)
        lib = _lib.load()
        nbytes = lib.vc_rcnn_loss_ws_bytes(K)
        ws = torch.empty((max(1, nbytes),), dtype=torch.uint8, device=dev)
        check(lib.vc_rcnn_loss(ctypes.addressof(table), K, cfg.beta, host_f64(cfg.code_weights), cfg.cls_weight,
                               cfg.reg_weight, cfg.corner_weight, int(cfg.corner), stats.data_ptr(), ws.data_ptr(), nbytes,
                               ops._stream()), 'vc_rcnn_loss')
        ctx.save_for_backward(*grads)
        ctx.shapes = [p.shape for p in preds]
        ctx.mark_non_differentiable(stats)
        return stats[K * 4].clone(), stats

    @staticmethod
    def backward(ctx, grad_loss, grad_stats):
        return (None, None, None) + tuple((g * grad_loss).view(s) for g, s in zip(ctx.saved_tensors, ctx.shapes))


def rcnn_loss(branches, cfg):
    """branches: [(targets dict with rcnn_cls [n, 1], rcnn_reg [n, 7], rois [B, R, 7], gt_of_rois (canonical) and
    gt_of_rois_src [B, R, ldg], reg_valid_mask [B, R], rcnn_cls_labels [B, R]; weight), ...] (n = B * R, at most 18),
    cfg = RCNNLossConfig, all CUDA -> (loss: 0-d tensor = rcnn_loss, stats: detached fp32 [K * 4 + 1] = per branch
    (cls, reg, corner, bb), then the weighted total).  No host read: capturable."""
    if not 1 <= len(branches) <= MAX_BRANCHES:
        raise ValueError(f'rcnn_loss: {len(branches)} branches (1..{MAX_BRANCHES})')
    preds = []
    for t, _ in branches:
        preds += [t['rcnn_cls'], t['rcnn_reg']]
    return _RCNNLoss.apply(cfg, [w for _, w in branches], [t for t, _ in branches], *preds)


def head_anchors(anchors):
    """the reference's `torch.cat(self.anchors, dim=-3).view(-1, 7)` (or self.anchors viewed) as [N, 7] fp32.  For the
    masked anchor sets AnchorHeadSingle.forward makes ([1, L, sizes, rotations, 7]) that is ordered_anchors' order, the
    one the target assignment writes; a full map with several sets ([1, H, W, sizes, rotations, 7]) is concatenated as
    the loss does."""
    if isinstance(anchors, (list, tuple)):
        if len(anchors) == 1 or all(a.dim() == 5 for a in anchors):
            return ordered_anchors(anchors)[0]
        return torch.cat(list(anchors), dim=-3).reshape(-1, 7).float().contiguous()
    return anchors.reshape(-1, anchors.shape[-1]).float().contiguous()


def anchor_head_get_loss(self):
    """AnchorHeadTemplate.get_loss (bound by reference_env.install(use_fused_losses=True)): the same (rpn_loss, tb_dict);
    the tb floats come from one device-to-host copy."""
    cfg = getattr(self, '_fused_rpn_loss_cfg', None)
    if cfg is None:
        cfg = self._fused_rpn_loss_cfg = RPNLossConfig(self.model_cfg, self.num_class)
    d = self.forward_ret_dict
    dir_preds = d.get('dir_cls_preds', None)
    loss, stats = rpn_loss(d['cls_preds'], d['box_preds'], dir_preds, d['box_cls_labels'], d['box_reg_targets'],
                           head_anchors(self.anchors), cfg)
    v = stats.cpu().tolist()
    tb_dict = {'rpn_loss_cls': v[0], 'rpn_loss_loc': v[1]}
    if dir_preds is not None:
        tb_dict['rpn_loss_dir'] = v[2]
    tb_dict['rpn_loss'] = v[3]
    return loss, tb_dict


def roi_head_branches(forward_ret_dict):
    """[(targets dict, weight)] in the reference's order: for each stage i < 6, targets_dict{i} (1), _pi{i} (0.5),
    _p{i} (0.5), those present"""
    return [(forward_ret_dict[key + str(i)], w) for i in range(6) for key, w in BRANCH_KEYS
            if key + str(i) in forward_ret_dict]


def roi_head_get_loss(self, tb_dict=None):
    """RoIHeadTemplate.get_loss (bound by reference_env.install(use_fused_losses=True)): the same (rcnn_loss, tb_dict);
    the tb float comes from one device-to-host copy."""
    tb_dict = {} if tb_dict is None else tb_dict
    cfg = getattr(self, '_fused_rcnn_loss_cfg', None)
    if cfg is None:
        cfg = self._fused_rcnn_loss_cfg = RCNNLossConfig(self.model_cfg)
    branches = roi_head_branches(self.forward_ret_dict)
    if not branches:
        raise ValueError(f'roi_head_get_loss: no targets_dict* in forward_ret_dict ({_REF_RCNN} fails there too)')
    loss, stats = rcnn_loss(branches, cfg)
    tb_dict['rcnn_loss'] = stats.cpu().tolist()[-1]
    return loss, tb_dict
