"""numpy float32 restatement of the RoI target sampling (rules 1-6 of virconv_b200/csrc/roi_targets.cu): what
ProposalTargetLayer.forward (SAMPLE_ROI_BY_EACH_CLASS True, CLS_SCORE_TYPE roi_iou_x) and the canonical transform of
RoIHeadTemplate.assign_targets compute, with the reference's host draws taken from given uniforms.  The 3-D IoU is the
caller's: `iou(roi_boxes [M, 7], gt_boxes [n, 7]) -> [M, n] float32` (oracle/iou3d.py in float64 rounded to fp32, or
the library's own vc_boxes_iou3d matrix)."""
from __future__ import annotations

import numpy as np

F32 = np.float32
TWO_PI = F32(2 * np.pi)


def trimmed_count(gt):
    """rule 1: rows dropped from the end while their sum over all columns is 0; row 0 stays"""
    k = len(gt) - 1
    while k > 0 and gt[k].sum(dtype=F32) == 0:
        k -= 1
    return k + 1


def draw(u, n):
    """rule 4: min(int(double(u) * n), n - 1), elementwise"""
    return np.minimum(np.floor(np.asarray(u, np.float64) * n).astype(np.int64), n - 1)


def remainder(a, b):
    """torch.remainder for float32 (fmod, plus the divisor when the signs differ)"""
    a = np.asarray(a, F32)
    m = np.fmod(a, F32(b))
    return np.where((m != 0) & ((F32(b) < 0) != (m < 0)), (m + F32(b)).astype(F32), m).astype(F32)


def match(rois, roi_labels, gt, iou):
    """rule 2 for one scene (gt already trimmed) -> ov [M] fp32, asg [M] int64"""
    M = len(rois)
    ov, asg = np.zeros(M, F32), np.zeros(M, np.int64)
    cls = gt[:, -1].astype(np.int64)
    mat = np.asarray(iou(rois[:, :7], gt[:, :7]), F32) if M and len(gt) else np.zeros((M, len(gt)), F32)
    for i in range(M):
        cand = np.nonzero(cls == roi_labels[i])[0]
        if len(cand):
            v = mat[i, cand]
            j = int(np.argmax(v))           # first maximum
            ov[i], asg[i] = v[j], cand[j]
    return ov, asg


def _bg(hard, easy, n, u_bg, ratio):
    if len(hard) and len(easy):
        h = min(int(n * ratio), len(hard))
        return np.concatenate([hard[draw(u_bg[:h], len(hard))], easy[draw(u_bg[h:n], len(easy))]])
    if len(hard):
        return hard[draw(u_bg[:n], len(hard))]
    return easy[draw(u_bg[:n], len(easy))]


def subsample(ov, gcls, cfg, u_fg, u_bg):
    """rules 3-4 for one scene -> sampled RoI indices [R], or None for the neither-branch"""
    lo = F32(cfg.CLS_BG_THRESH_LO)
    fg = np.zeros(len(ov), bool)
    hard = np.zeros(len(ov), bool)
    for i in range(len(cfg.CLS_FG_THRESH)):
        m = gcls == F32(i + 1)
        fg |= (ov >= F32(min(cfg.REG_FG_THRESH[i], cfg.CLS_FG_THRESH[i]))) & m
    for i in range(len(cfg.REG_FG_THRESH)):
        m = gcls == F32(i + 1)
        hard |= (ov < F32(cfg.REG_FG_THRESH[i])) & (ov >= lo) & m
    fg, hard, easy = np.nonzero(fg)[0], np.nonzero(hard)[0], np.nonzero(ov < lo)[0]
    R = int(cfg.ROI_PER_IMAGE)
    F = int(np.round(cfg.FG_RATIO * cfg.ROI_PER_IMAGE))
    nf, nb = len(fg), len(hard) + len(easy)
    if nf > 0 and nb > 0:
        kf = min(F, nf)
        order = np.argsort(np.asarray(u_fg[:nf], F32), kind='stable')[:kf]
        return np.concatenate([fg[order], _bg(hard, easy, R - kf, u_bg, cfg.HARD_BG_RATIO)])
    if nf > 0:
        return fg[draw(u_fg[:R], nf)]
    if nb > 0:
        return _bg(hard, easy, R, u_bg, cfg.HARD_BG_RATIO)
    return None


def labels(ov, gcls, cfg, u_hs, B):
    """rule 5 over [B, R] -> reg_valid_mask int64, rcnn_cls_labels fp32"""
    reg = np.zeros(ov.shape, np.int64)
    for i in range(len(cfg.REG_FG_THRESH)):
        m = gcls == F32(i + 1)
        t = F32(cfg.REG_FG_THRESH[i])
        this = ((ov > t) & m).astype(np.int64)
        if cfg.get('ENABLE_HARD_SAMPLING', False):
            per = int(1 / cfg.HARD_SAMPLING_RATIO[i])
            sel = np.zeros(ov.shape, bool)
            sel[range(int(draw(u_hs[i], per)), B, per)] = True
            this += ((ov < t) & (ov > F32(cfg.HARD_SAMPLING_THRESH[i])) & m & sel).astype(np.int64)
        reg += this
    cls = np.zeros(ov.shape, F32)
    for i in range(len(cfg.CLS_BG_THRESH)):
        m = gcls == F32(i + 1)
        fg_t, bg_t = F32(cfg.CLS_FG_THRESH[i]), F32(cfg.CLS_BG_THRESH[i])
        inv = F32(1.0) / F32(cfg.CLS_FG_THRESH[i] - cfg.CLS_BG_THRESH[i])
        v = np.where(ov > fg_t, F32(1), np.where(ov < bg_t, F32(0), ((ov - bg_t) * inv).astype(F32))).astype(F32)
        cls[m] = v[m]
    return reg, cls


def canonical(rois, gt_src):
    """rule 6 over [..., C]: the canonical transform of the gathered GT rows"""
    out = gt_src.astype(F32).copy()
    x, y, z = (gt_src[..., k] - rois[..., k] for k in range(3))
    ry = remainder(rois[..., 6], TWO_PI)
    c, s = np.cos(-ry).astype(F32), np.sin(-ry).astype(F32)
    out[..., 0] = x * c + y * -s
    out[..., 1] = x * s + y * c
    out[..., 2] = z
    h = remainder(gt_src[..., 6] - ry, TWO_PI)
    opp = (h > F32(np.pi * 0.5)) & (h < F32(np.pi * 1.5))
    h = np.where(opp, remainder(h + F32(np.pi), TWO_PI), h)
    h = np.where(h > F32(np.pi), (h - TWO_PI).astype(F32), h)
    out[..., 6] = np.clip(h, F32(-np.pi / 2), F32(np.pi / 2))
    return out


def sample(cfg, rois, roi_scores, roi_labels, gt, u_fg, u_bg, u_hs, iou):
    """all scenes -> dict of the kernel's outputs (numpy) plus 'sampled' [B, R] RoI indices (-1 in a neither-branch
    scene, whose rows are zero, as is its count in 'status')"""
    rois, gt = np.asarray(rois, F32), np.asarray(gt, F32)
    B, R = rois.shape[0], int(cfg.ROI_PER_IMAGE)
    out = {'rois': np.zeros((B, R, rois.shape[-1]), F32), 'gt_of_rois_src': np.zeros((B, R, gt.shape[-1]), F32),
           'gt_iou_of_rois': np.zeros((B, R), F32), 'roi_scores': np.zeros((B, R), F32),
           'roi_labels': np.zeros((B, R), np.int64), 'sampled': np.full((B, R), -1, np.int64)}
    ok = np.zeros(B, bool)
    for b in range(B):
        g = gt[b, :trimmed_count(gt[b])] if gt.shape[1] else np.zeros((1, gt.shape[-1]), F32)
        ov, asg = match(rois[b], np.asarray(roi_labels[b]), g, iou)
        idx = subsample(ov, g[asg, -1], cfg, u_fg[b], u_bg[b])
        if idx is None:
            continue
        ok[b] = True
        out['sampled'][b] = idx
        out['rois'][b] = rois[b, idx]
        out['gt_of_rois_src'][b] = g[asg[idx]]
        out['gt_iou_of_rois'][b] = ov[idx]
        out['roi_scores'][b] = np.asarray(roi_scores[b], F32)[idx]
        out['roi_labels'][b] = np.asarray(roi_labels[b])[idx]
    reg, cls = labels(out['gt_iou_of_rois'], out['gt_of_rois_src'][..., -1], cfg, u_hs, B)
    out['reg_valid_mask'], out['rcnn_cls_labels'] = reg * ok[:, None], cls * ok[:, None]
    out['gt_of_rois'] = canonical(out['rois'], out['gt_of_rois_src'])
    out['status'] = int((~ok).sum())
    return out
