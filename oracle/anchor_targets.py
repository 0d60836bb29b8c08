"""numpy float32 restatement of csrc/anchor_targets.cu (rules 0-5 of its header): the RPN's anchor mask
(AnchorHeadSingle.get_anchor_mask) and AxisAlignedTargetAssigner.assign_targets with POS_FRACTION < 0, written the way the
reference writes them (dense IoU matrix per scene and anchor set, numpy argmax, boolean masks), with the GPU's
division-by-scalar (a multiply by the fp32 reciprocal) in limit_period.  Test infrastructure only."""
from __future__ import annotations

import numpy as np

F = np.float32
PI = F(np.pi)
INV_PI = F(1) / PI
PI4 = F(np.pi / 4)


def anchor_mask(points, min_x, min_y, inv_stride, H, W):
    """points [Np, >= 3] (column 1 = x, 2 = y) -> bool [H, W] (rule 0: the reference's coarse map, argwhere, the 20 x 20
    window list and numpy's wrap of negative indices)"""
    h10, w10 = H // 10, W // 10
    p = np.asarray(points, F)
    cx = ((p[:, 1] - F(min_x)) * F(inv_stride)).astype(np.int64)
    cy = ((p[:, 2] - F(min_y)) * F(inv_stride)).astype(np.int64)
    cx, cy = np.minimum(cx, w10 - 1), np.minimum(cy, h10 - 1)
    keep = (cx >= -w10) & (cy >= -h10)
    coarse = np.zeros((h10, w10), bool)
    coarse[cy[keep], cx[keep]] = True
    idx = np.argwhere(coarse) * 10
    ii, jj = np.meshgrid(np.arange(-10, 10), np.arange(-10, 10), indexing='ij')
    mask = np.zeros((H, W), bool)
    mask[(idx[:, None, 0] + ii.ravel()[None]).ravel(), (idx[:, None, 1] + jj.ravel()[None]).ravel()] = True
    return mask


def anchors_from_shifts(x_shifts, y_shifts, bottom_heights, sizes, rotations):
    """AnchorGenerator.generate_anchors for one anchor set from its 1-D shift vectors -> [Z, Y, X, n_size, n_rot, 7]"""
    xs, ys = np.asarray(x_shifts, F), np.asarray(y_shifts, F)
    zs, sizes, rots = np.asarray(bottom_heights, F), np.asarray(sizes, F).reshape(-1, 3), np.asarray(rotations, F)
    X, Y, Z, ns, nr = len(xs), len(ys), len(zs), len(sizes), len(rots)
    a = np.zeros((Z, Y, X, ns, nr, 7), F)
    a[..., 0] = xs[None, None, :, None, None]
    a[..., 1] = ys[None, :, None, None, None]
    a[..., 2] = zs[:, None, None, None, None]
    a[..., 3:6] = sizes[None, None, None, :, None, :]
    a[..., 6] = rots
    a[..., 2] += a[..., 5] / F(2)
    return a


def ordered(all_anchors):
    """rule 5: each set viewed as (shape[0], shape[1], -1, 7), concatenated per location -> (anchors [N, 7], set [N])"""
    L = all_anchors[0].shape[0] * all_anchors[0].shape[1]
    parts = [np.asarray(a, F).reshape(L, -1, 7) for a in all_anchors]
    sid = np.concatenate([np.full((L, p.shape[1]), s, np.int32) for s, p in enumerate(parts)], 1).reshape(-1)
    return np.concatenate(parts, 1).reshape(-1, 7), sid


def nearest_bev(boxes):
    """rule 2: [n, 7] -> (x1, y1, x2, y2) [n, 4], area [n]"""
    b = np.asarray(boxes, F)
    h = b[:, 6]
    r = np.abs(h - np.floor(h * INV_PI + F(0.5)) * PI)
    keep = r < PI4
    d = np.where(keep[:, None], b[:, [3, 4]], b[:, [4, 3]]) / F(2)
    bev = np.concatenate([b[:, 0:2] - d, b[:, 0:2] + d], 1)
    return bev, (bev[:, 2] - bev[:, 0]) * (bev[:, 3] - bev[:, 1])


def iou_nearest(a, b):
    (ba, aa), (bb, ab) = nearest_bev(a), nearest_bev(b)
    xl = np.maximum(np.minimum(ba[:, None, 2], bb[None, :, 2]) - np.maximum(ba[:, None, 0], bb[None, :, 0]), F(0))
    yl = np.maximum(np.minimum(ba[:, None, 3], bb[None, :, 3]) - np.maximum(ba[:, None, 1], bb[None, :, 1]), F(0))
    inter = xl * yl
    return inter / np.maximum(aa[:, None] + ab[None, :] - inter, F(1e-6))


def encode(g, a):
    """rule 4 (ResidualCoder.encode_torch), fp32"""
    g, a = np.array(g, F), np.array(a, F)
    a[:, 3:6] = np.maximum(a[:, 3:6], F(1e-5))
    g[:, 3:6] = np.maximum(g[:, 3:6], F(1e-5))
    diag = np.sqrt(a[:, 3] * a[:, 3] + a[:, 4] * a[:, 4])
    return np.stack([(g[:, 0] - a[:, 0]) / diag, (g[:, 1] - a[:, 1]) / diag, (g[:, 2] - a[:, 2]) / a[:, 5],
                     np.log(g[:, 3] / a[:, 3]), np.log(g[:, 4] / a[:, 4]), np.log(g[:, 5] / a[:, 5]), g[:, 6] - a[:, 6]],
                    1).astype(F)


def trimmed_count(gt):
    """rule 1: rows kept of one scene's [M, C] GT"""
    cnt = len(gt) - 1
    while cnt > 0 and gt[cnt, :-1].sum() == 0:
        cnt -= 1
    return cnt + 1


def assign(anchors, anchor_set, gt, class_names, anchor_class_names, matched, unmatched):
    """anchors [N, 7], anchor_set [N] (ordered()), gt [B, M, C] -> labels [B, N] int32, targets [B, N, 7], reg_weights,
    gt_ious [B, N] fp32 (rules 1, 3, 4)"""
    anchors, gt = np.asarray(anchors, F), np.asarray(gt, F)
    B, N = gt.shape[0], anchors.shape[0]
    labels = np.zeros((B, N), np.int32)
    targets = np.zeros((B, N, 7), F)
    reg = np.zeros((B, N), F)
    ious = np.full((B, N), -0.0, F)
    names = np.array(class_names)
    for b in range(B):
        g = gt[b][:trimmed_count(gt[b])]
        cls = g[:, -1].astype(np.int32)
        for s, name in enumerate(anchor_class_names):
            rows = np.nonzero(anchor_set == s)[0]
            sel = np.array([-len(names) <= c - 1 < len(names) and names[c - 1] == name for c in cls], bool)
            tg, tc = g[sel], cls[sel]
            if len(tg) == 0 or len(rows) == 0:
                continue
            a = anchors[rows]
            m = iou_nearest(a, tg[:, :7])
            arg = m.argmax(1)
            mx = m[np.arange(len(rows)), arg]
            col = m.max(0)
            col[col == 0] = -1
            forced = (m == col[None]).any(1)
            lab = np.full(len(rows), -1, np.int32)
            lab[mx >= F(matched[s])] = tc[arg][mx >= F(matched[s])]
            lab[mx < F(unmatched[s])] = 0
            lab[forced] = tc[arg][forced]
            labels[b, rows] = lab
            ious[b, rows] = mx
            fg = lab > 0
            t = np.zeros((len(rows), 7), F)
            if fg.any():
                t[fg] = encode(tg[arg[fg], :7], a[fg])
            targets[b, rows] = t
            reg[b, rows] = fg.astype(F)
    return labels, targets, reg, ious
