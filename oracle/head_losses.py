"""Float64 numpy restatement of the detection losses of csrc/head_losses.cu (rules R1-R7, C1-C6) and of their
closed-form gradients.  It follows the reference's dtypes: the RPN's classification and box weights are the fp32
1 / n that `positives.float() / clamp(...)` makes; everything else is float64.

    rpn(cls, box, dir, labels, targets, anchors, cfg)  -> (losses [4], g_cls, g_box, g_dir)
    rcnn(branches, cfg)                                -> (losses [K * 4 + 1], [(g_cls, g_reg), ...])
cfg: an object with the attributes of virconv_b200.head_losses.RPNLossConfig / RCNNLossConfig."""
from __future__ import annotations

import numpy as np

TWO_PI = 2 * np.pi
TEMPLATE = np.array([[1, 1, -1], [1, -1, -1], [-1, -1, -1], [-1, 1, -1],
                     [1, 1, 1], [1, -1, 1], [-1, -1, 1], [-1, 1, 1]], np.float64) / 2


def smooth_l1(d, beta):
    """value and d value / d d (sign(0) = 0, the where's branch as written)"""
    n = np.abs(d)
    small = n < beta
    val = np.where(small, 0.5 * n ** 2 / beta, n - 0.5 * beta)
    grad = np.where(small, n / beta, 1.0) * np.sign(d)
    return val, grad


def rpn(cls, box, dir_, labels, targets, anchors, cfg):
    B = cls.shape[0]
    C = cfg.num_class
    cls = np.asarray(cls, np.float64).reshape(B, -1, C)
    N = cls.shape[1]
    box = np.asarray(box, np.float64).reshape(B, N, 7)
    tgt = np.asarray(targets, np.float64).reshape(B, N, 7)
    y = np.asarray(labels).reshape(B, N).astype(np.int64)
    npos = np.maximum((y > 0).sum(1, keepdims=True), 1)
    wpos = (np.float32(1) / npos.astype(np.float32)).astype(np.float64)          # R1
    # R2-R4
    wc = np.where(y >= 0, wpos, 0.0)
    tcls = np.where(y > 0, 1 if C == 1 else y, 0)
    t = (tcls[..., None] == np.arange(1, C + 1)).astype(np.float64)
    p = 1.0 / (1.0 + np.exp(-cls))
    aw = t * cfg.alpha + (1 - t) * (1 - cfg.alpha)
    pt = t * (1.0 - p) + (1.0 - t) * p
    fw = aw * pt ** cfg.gamma
    ex = np.exp(-np.abs(cls))
    bce = np.maximum(cls, 0) - cls * t + np.log1p(ex)
    l_cls = (fw * bce * wc[..., None]).sum()
    dfw = aw * cfg.gamma * pt ** (cfg.gamma - 1) if cfg.gamma != 0 else 0.0
    dpt = (1 - 2 * t) * ((1 - p) * p)
    dbce = (cls >= 0).astype(np.float64) - t - np.sign(cls) * (ex / (1 + ex))
    g_cls = (dfw * dpt * bce + fw * dbce) * wc[..., None] * (cfg.cls_weight / B)
    # R5
    wr = np.where(y > 0, wpos, 0.0)
    xi, ti = box.copy(), tgt.copy()
    dxi, dti = np.ones_like(box), np.zeros_like(box)
    x6, t6 = box[..., 6], tgt[..., 6]
    with np.errstate(invalid='ignore'):
        xi[..., 6] = np.sin(x6) * np.cos(t6)
        ti[..., 6] = np.cos(x6) * np.sin(t6)
        dxi[..., 6] = np.cos(x6) * np.cos(t6)
        dti[..., 6] = -np.sin(x6) * np.sin(t6)
    nan = np.isnan(ti)
    ti = np.where(nan, xi, ti)
    dti = np.where(nan, dxi, dti)
    cw = np.asarray(cfg.code_weights, np.float64)
    val, gd = smooth_l1((xi - ti) * cw, cfg.beta)
    l_loc = (val * wr[..., None]).sum()
    g_box = gd * cw * (dxi - dti) * wr[..., None] * (cfg.loc_weight / B)
    # R6
    l_dir, g_dir = 0.0, None
    if dir_ is not None:
        nb = cfg.num_dir_bins
        z = np.asarray(dir_, np.float64).reshape(B, N, nb)
        wd = np.where(y > 0, 1.0 / npos, 0.0)
        v = (tgt[..., 6] + np.asarray(anchors, np.float64)[None, :, 6]) - cfg.dir_offset
        off = v - np.floor(v / TWO_PI) * TWO_PI
        b = np.clip(np.floor(off / (TWO_PI / nb)), 0, nb - 1).astype(np.int64)
        m = z.max(-1, keepdims=True)
        e = np.exp(z - m)
        se = e.sum(-1, keepdims=True)
        lse = m[..., 0] + np.log(se[..., 0])
        l_dir = ((lse - np.take_along_axis(z, b[..., None], -1)[..., 0]) * wd).sum()
        g_dir = (e / se - (np.arange(nb) == b[..., None])) * wd[..., None] * (cfg.dir_weight / B)
    cls_v, loc_v = l_cls / B * cfg.cls_weight, l_loc / B * cfg.loc_weight
    dir_v = l_dir / B * cfg.dir_weight if dir_ is not None else 0.0
    return np.array([cls_v, loc_v, dir_v, cls_v + loc_v + dir_v]), g_cls, g_box, g_dir


def encode(g, a):
    """ResidualCoder.encode_torch, sizes clamped at 1e-5"""
    a, g = a.copy(), g.copy()
    a[:, 3:6] = np.maximum(a[:, 3:6], 1e-5)
    g[:, 3:6] = np.maximum(g[:, 3:6], 1e-5)
    diag = np.sqrt(a[:, 3] ** 2 + a[:, 4] ** 2)
    return np.stack([(g[:, 0] - a[:, 0]) / diag, (g[:, 1] - a[:, 1]) / diag, (g[:, 2] - a[:, 2]) / a[:, 5],
                     np.log(g[:, 3] / a[:, 3]), np.log(g[:, 4] / a[:, 4]), np.log(g[:, 5] / a[:, 5]), g[:, 6] - a[:, 6]], 1)


def decode(t, a):
    diag = np.sqrt(a[:, 3] ** 2 + a[:, 4] ** 2)
    return np.stack([t[:, 0] * diag + a[:, 0], t[:, 1] * diag + a[:, 1], t[:, 2] * a[:, 5] + a[:, 2],
                     np.exp(t[:, 3]) * a[:, 3], np.exp(t[:, 4]) * a[:, 4], np.exp(t[:, 5]) * a[:, 5], t[:, 6] + a[:, 6]], 1)


def corners(b):
    """[n, 8, 3] corners of boxes [n, 7] (box_utils.boxes_to_corners_3d)"""
    loc = b[:, None, 3:6] * TEMPLATE[None]
    c, s = np.cos(b[:, 6])[:, None], np.sin(b[:, 6])[:, None]
    return np.stack([loc[..., 0] * c - loc[..., 1] * s + b[:, None, 0], loc[..., 0] * s + loc[..., 1] * c + b[:, None, 1],
                     loc[..., 2] + b[:, None, 2]], -1)


def pick_min(a, b):
    return np.where(a < b, 1.0, np.where(a == b, 0.5, 0.0))


def pick_max(a, b):
    return np.where(a > b, 1.0, np.where(a == b, 0.5, 0.0))


def limit(a):
    a = a - np.floor(a / TWO_PI) * TWO_PI
    a = np.where(a > np.pi, a - TWO_PI, a)
    return np.where(a < -np.pi, a + TWO_PI, a)


def iou_1d(x, w, y, l):
    hi1, lo1, hi2, lo2 = x + w * 0.5, x - w * 0.5, y + l * 0.5, y - l * 0.5
    ov_raw = np.minimum(hi1, hi2) - np.maximum(lo1, lo2)
    al_raw = np.maximum(hi1, hi2) - np.minimum(lo1, lo2)
    ov, al = np.maximum(ov_raw, 0), np.maximum(al_raw, 0)
    d_ov, d_al = 1 / al, -ov / al ** 2
    p_ov, p_al = (ov_raw >= 0).astype(np.float64), (al_raw >= 0).astype(np.float64)
    d_hi = d_ov * p_ov * pick_min(hi1, hi2) + d_al * p_al * pick_max(hi1, hi2)
    d_lo = -d_ov * p_ov * pick_max(lo1, lo2) - d_al * p_al * pick_min(lo1, lo2)
    return ov / al, d_hi + d_lo, (d_hi - d_lo) * 0.5


def rcnn_branch(t, cfg):
    """one branch (a dict of numpy arrays: rcnn_cls, rcnn_reg, rois, gt_of_rois, gt_of_rois_src, reg_valid_mask,
    rcnn_cls_labels) -> ((cls, reg, corner, bb), g_cls [n], g_reg [n, 7]) without the branch weight"""
    x = np.asarray(t['rcnn_cls'], np.float64).reshape(-1)
    n = x.shape[0]
    r = np.asarray(t['rcnn_reg'], np.float64).reshape(n, 7)
    roi = np.asarray(t['rois'], np.float64).reshape(n, -1)[:, :7]
    gt = np.asarray(t['gt_of_rois'], np.float64).reshape(n, -1)[:, :7]
    src = np.asarray(t['gt_of_rois_src'], np.float64).reshape(n, -1)[:, :7]
    fgm = np.asarray(t['reg_valid_mask']).reshape(-1) > 0
    y = np.asarray(t['rcnn_cls_labels'], np.float64).reshape(-1)
    fg, nv = int(fgm.sum()), int((y >= 0).sum())
    # C2
    p = 1 / (1 + np.exp(-x))
    with np.errstate(divide='ignore'):
        lp, l1p = np.maximum(np.log(p), -100), np.maximum(np.log(1 - p), -100)
    vm = (y >= 0).astype(np.float64)
    cls = (((y - 1) * l1p - y * lp) * vm).sum() / max(nv, 1) * cfg.cls_weight
    q = (1 - p) * p
    g_cls = (p - y) / np.maximum(q, 1e-12) * q * vm * (cfg.cls_weight / max(nv, 1))
    # C3
    anc = np.zeros((n, 7))
    anc[:, 3:6] = roi[:, 3:6]
    tg = encode(gt, anc)
    nan = np.isnan(tg)
    cw = np.asarray(cfg.code_weights, np.float64)
    val, gd = smooth_l1((r - np.where(nan, r, tg)) * cw, cfg.beta)
    reg = (val * fgm[:, None]).sum() / max(fg, 1) * cfg.reg_weight
    g_reg = np.where(nan, 0.0, gd * cw) * fgm[:, None] * (cfg.reg_weight / max(fg, 1))
    # C4
    corner = 0.0
    f = np.nonzero(fgm)[0]
    if cfg.corner and fg > 0:
        a4 = anc[f].copy()
        a4[:, 6] = roi[f, 6]
        pb = decode(r[f], a4)
        c0, s0 = np.cos(roi[f, 6]), np.sin(roi[f, 6])
        cx, cy = pb[:, 0].copy(), pb[:, 1].copy()
        pb[:, 0] = cx * c0 - cy * s0 + roi[f, 0]
        pb[:, 1] = cx * s0 + cy * c0 + roi[f, 1]
        pb[:, 2] = pb[:, 2] + roi[f, 2]
        gs = src[f]
        gf = gs.copy()
        gf[:, 6] = gs[:, 6] + np.pi
        pc, gc, fc = corners(pb), corners(gs), corners(gf)
        d1, d2 = pc - gc, pc - fc
        n1, n2 = np.linalg.norm(d1, axis=-1), np.linalg.norm(d2, axis=-1)
        dist = np.minimum(n1, n2)
        lv, dl = smooth_l1(dist, 1.0)
        corner = lv.mean(1).mean() * cfg.corner_weight
        with np.errstate(invalid='ignore', divide='ignore'):
            u1 = np.where(n1[..., None] == 0, 0.0, d1 / n1[..., None])
            u2 = np.where(n2[..., None] == 0, 0.0, d2 / n2[..., None])
        gp = (pick_min(n1, n2) * dl)[..., None] * u1 + (pick_min(n2, n1) * dl)[..., None] * u2   # [fg, 8, 3]
        ch, sh = np.cos(pb[:, 6])[:, None], np.sin(pb[:, 6])[:, None]
        lx, ly = pb[:, None, 3] * TEMPLATE[None, :, 0], pb[:, None, 4] * TEMPLATE[None, :, 1]
        gC = gp.sum(1)
        gdx = ((gp[..., 0] * ch + gp[..., 1] * sh) * TEMPLATE[None, :, 0]).sum(1)
        gdy = ((-gp[..., 0] * sh + gp[..., 1] * ch) * TEMPLATE[None, :, 1]).sum(1)
        gdz = (gp[..., 2] * TEMPLATE[None, :, 2]).sum(1)
        gh = (gp[..., 0] * -(lx * sh + ly * ch) + gp[..., 1] * (lx * ch - ly * sh)).sum(1)
        gxl, gyl = gC[:, 0] * c0 + gC[:, 1] * s0, -gC[:, 0] * s0 + gC[:, 1] * c0
        diag = np.sqrt(roi[f, 3] ** 2 + roi[f, 4] ** 2)
        s = cfg.corner_weight / fg / 8
        g_reg[f] += np.stack([gxl * diag, gyl * diag, gC[:, 2] * roi[f, 5], gdx * pb[:, 3], gdy * pb[:, 4],
                              gdz * pb[:, 5], gh], 1) * s
    # C5
    bb = 0.0
    if fg > 0:
        pb = decode(r[f], anc[f])
        g = gt[f]
        iu, gx, gw = zip(*[iou_1d(pb[:, a], pb[:, a + 3], g[:, a], g[:, a + 3]) for a in range(3)])
        dlt = limit(pb[:, 6]) - limit(g[:, 6])
        ia = 1 - np.abs(np.sin(dlt))
        dia = -np.sign(np.sin(dlt)) * np.cos(dlt)
        da = pb[:, 6] - g[:, 6]
        af = 1.25 * (1 - np.abs(np.cos(da)))
        daf = 1.25 * np.sign(np.cos(da)) * np.sin(da)
        cd = ((g[:, :3] - pb[:, :3]) ** 2).sum(1)
        bb = ((1 - iu[0] * iu[1] * iu[2] * ia + af + cd) * 1.5).sum() / (fg + 1)
        others = [iu[1] * iu[2] * ia, iu[0] * iu[2] * ia, iu[0] * iu[1] * ia, iu[0] * iu[1] * iu[2]]
        diag = np.sqrt(roi[f, 3] ** 2 + roi[f, 4] ** 2)
        sc = [diag, diag, roi[f, 5]]
        s = 1.5 / (fg + 1)
        for a in range(3):
            g_reg[f, a] += (-others[a] * gx[a] + 2 * (pb[:, a] - g[:, a])) * sc[a] * s
            g_reg[f, a + 3] += -others[a] * gw[a] * pb[:, a + 3] * s
        g_reg[f, 6] += (-others[3] * dia + daf) * s
    return np.array([cls, reg, corner, bb]), g_cls.reshape(np.shape(t['rcnn_cls'])), g_reg


def rcnn(branches, cfg):
    """branches: [(dict of numpy arrays, weight)] -> (losses [K * 4 + 1], [(g_cls, g_reg) of d total / d preds])"""
    out, grads, tot = [], [], 0.0
    for t, w in branches:
        v, gc, gr = rcnn_branch(t, cfg)
        out.append(v)
        grads.append((gc * w, gr * w))
        tot += w * v.sum()
    return np.concatenate(out + [np.array([tot])]), grads
