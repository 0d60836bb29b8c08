"""Restatements of csrc/box_decode.cu (rules R1-R3 of its header).  Test infrastructure only.

  * numpy in float64 (the default) or float32 (`dtype=np.float32`, each operation rounding once as torch's elementwise
    kernels round it): anchor_decode, roi_decode, xtrans, and the closed-form gradients anchor_decode_grad /
    roi_decode_grad with respect to box_preds;
  * torch, on any device and dtype, following the reference's own control flow (the per-scene loops, the `if enable`
    host read, the 3 x 3 matmul): torch_anchor_decode, torch_roi_decode, torch_roi_x_trans, torch_roi_score_trans,
    torch_pred_x_trans.  profiles/microbench_box_decode.py times them as the reference path, and the GPU tests
    differentiate the float64 ones with torch.autograd.

`div` selects how limit_period divides by the period in float32: True as torch's CPU kernel does (a true division), False
as its CUDA kernel does for a CPU scalar (a multiplication by the float32 reciprocal, the kernel's rule)."""
from __future__ import annotations

import numpy as np
import torch

F64 = np.float64


def _decode(t, a, dt):
    """ResidualCoder.decode_torch: t, a [..., 7] -> [..., 7] (box_coder.cuh residual_decode)"""
    diag = np.sqrt(a[..., 3] * a[..., 3] + a[..., 4] * a[..., 4])
    g = np.empty(np.broadcast_shapes(t.shape, a.shape), dt)
    g[..., 0] = t[..., 0] * diag + a[..., 0]
    g[..., 1] = t[..., 1] * diag + a[..., 1]
    g[..., 2] = t[..., 2] * a[..., 5] + a[..., 2]
    for k in range(3, 6):
        g[..., k] = np.exp(t[..., k]) * a[..., k]
    g[..., 6] = t[..., 6] + a[..., 6]
    return g


def dir_labels(dir_cls):
    """torch.max(dim=-1)[1]: the first maximal bin, a NaN bin maximal (the first NaN)"""
    d = np.asarray(dir_cls)
    nan = np.isnan(d)
    return np.where(nan.any(-1), nan.argmax(-1), np.nanargmax(np.where(nan, -np.inf, d), -1))


def bin_quotient(val, period, limit_offset, dtype=F64, div=True):
    """limit_period's val / period + offset, before the floor"""
    dt = np.dtype(dtype).type
    val, p = np.asarray(val, dt), dt(period)
    q = val / p if div or dt is np.float64 else val * (dt(1) / p)
    return q + dt(limit_offset)


def anchor_decode(box, anchors, dir_cls=None, dir_offset=0.0, dir_limit_offset=0.0, period=np.pi, dtype=F64,
                  div=True):
    """R1: box [B, A, 7], anchors [A, 7], dir_cls [B, A, NB] or None -> [B, A, 7]"""
    dt = np.dtype(dtype).type
    t, a = np.asarray(box, dt), np.asarray(anchors, dt)[None]
    g = _decode(t, a, dt)
    if dir_cls is not None:
        label = dir_labels(dir_cls)
        off, p = dt(dir_offset), dt(period)
        val = g[..., 6] - off
        rot = val - np.floor(bin_quotient(val, period, dir_limit_offset, dt, div)) * p
        g[..., 6] = (rot + off) + p * label.astype(dt)
    return g


def anchor_decode_grad(grad, box, anchors, dtype=F64):
    """R2b for R1: d loss / d box_preds from grad = d loss / d boxes [B, A, 7]"""
    dt = np.dtype(dtype).type
    g, t, a = np.asarray(grad, dt), np.asarray(box, dt), np.asarray(anchors, dt)[None]
    diag = np.sqrt(a[..., 3] * a[..., 3] + a[..., 4] * a[..., 4])
    d = np.empty(np.broadcast_shapes(g.shape, a.shape), dt)
    d[..., 0] = g[..., 0] * diag
    d[..., 1] = g[..., 1] * diag
    d[..., 2] = g[..., 2] * a[..., 5]
    for k in range(3, 6):
        d[..., k] = (g[..., k] * a[..., k]) * np.exp(t[..., k])
    d[..., 6] = g[..., 6]
    return d


def _rotate(v, c, s):
    """[x y z] * [[c, s, 0], [-s, c, 0], [0, 0, 1]] in place on v[..., 0:3]"""
    x, y, z = v[..., 0].copy(), v[..., 1].copy(), v[..., 2].copy()
    zero = x.dtype.type(0)
    v[..., 0] = (x * c + y * (-s)) + z * zero
    v[..., 1] = (x * s + y * c) + z * zero
    v[..., 2] = (x * zero + y * zero) + z


def roi_decode(box, rois, dtype=F64):
    """R2: box [B * N, 7], rois [B, N, >= 7] -> [B, N, 7]"""
    dt = np.dtype(dtype).type
    r = np.asarray(rois, dt)[..., :7]
    B, N = r.shape[:2]
    local = r.copy()
    local[..., 0:3] = 0
    g = _decode(np.asarray(box, dt).reshape(B, N, 7), local, dt)
    _rotate(g, np.cos(r[..., 6]), np.sin(r[..., 6]))
    g[..., 0:3] += r[..., 0:3]
    return g


def roi_decode_grad(grad, box, rois, dtype=F64):
    """R2b for R2: d loss / d box_preds [B * N, 7] from grad = d loss / d boxes [B, N, 7]"""
    dt = np.dtype(dtype).type
    r = np.asarray(rois, dt)[..., :7]
    B, N = r.shape[:2]
    g = np.asarray(grad, dt).reshape(B, N, 7)
    t = np.asarray(box, dt).reshape(B, N, 7)
    c, s = np.cos(r[..., 6]), np.sin(r[..., 6])
    zero = dt(0)
    gx = (g[..., 0] * c + g[..., 1] * s) + g[..., 2] * zero
    gy = (g[..., 0] * (-s) + g[..., 1] * c) + g[..., 2] * zero
    gz = (g[..., 0] * zero + g[..., 1] * zero) + g[..., 2]
    diag = np.sqrt(r[..., 3] * r[..., 3] + r[..., 4] * r[..., 4])
    d = np.empty((B, N, 7), dt)
    d[..., 0], d[..., 1], d[..., 2] = gx * diag, gy * diag, gz * r[..., 5]
    for k in range(3, 6):
        d[..., k] = (g[..., k] * r[..., k]) * np.exp(t[..., k])
    d[..., 6] = g[..., 6]
    return d.reshape(B * N, 7)


def xtrans(boxes, tparam, from_stage, to_stage, dtype=F64):
    """R3: boxes [B, N, >= 7], tparam [B, R, 3] -> [B, N, same]; a stage None is skipped"""
    dt = np.dtype(dtype).type
    v = np.array(boxes, dt)
    p = np.asarray(tparam, dt)
    B = v.shape[0]

    def flip(f):
        on = ~(f == 0)
        v[on, :, 1] = -(v[on, :, 1] + dt(0))
        v[on, :, 6] = -(v[on, :, 6] + dt(0))

    def rotate(th):
        th = th[:, None]
        _rotate(v[..., 0:3], np.cos(th), np.sin(th))
        v[..., 6] = v[..., 6] + th

    if from_stage is not None:
        th, f, sc = p[:B, from_stage, 0], p[:B, from_stage, 1], p[:B, from_stage, 2]
        v[..., 0:6] = v[..., 0:6] / sc[:, None, None]
        flip(f)
        rotate(-th)
    if to_stage is not None:
        th, f, sc = p[:B, to_stage, 0], p[:B, to_stage, 1], p[:B, to_stage, 2]
        rotate(th)
        flip(f)
        v[..., 0:6] = v[..., 0:6] * sc[:, None, None]
    return v


def clamp_stage(i, R):
    while i >= R:
        i -= 1
    return i


# ---- the reference's control flow over torch ---------------------------------------------------------------------------
def torch_decode(box_encodings, anchors):
    """ResidualCoder.decode_torch (box_coder_utils.py:46-79) with 7 codes"""
    xa, ya, za, dxa, dya, dza, ra, *cas = torch.split(anchors, 1, dim=-1)
    xt, yt, zt, dxt, dyt, dzt, rt = torch.split(box_encodings, 1, dim=-1)
    diagonal = torch.sqrt(dxa ** 2 + dya ** 2)
    xg = xt * diagonal + xa
    yg = yt * diagonal + ya
    zg = zt * dza + za
    dxg = torch.exp(dxt) * dxa
    dyg = torch.exp(dyt) * dya
    dzg = torch.exp(dzt) * dza
    rg = rt + ra
    return torch.cat([xg, yg, zg, dxg, dyg, dzg, rg], dim=-1)


def torch_limit_period(val, offset, period):
    return val - torch.floor(val / period + offset) * period


def torch_anchor_decode(box, anchors, dir_cls=None, dir_offset=0.78539, dir_limit_offset=0.0, num_dir_bins=2):
    """generate_predicted_boxes' box branch: box [B, A, 7], anchors [A, 7], dir_cls [B, A, NB]"""
    B = box.shape[0]
    batch_anchors = anchors.view(1, -1, anchors.shape[-1]).repeat(B, 1, 1)
    out = torch_decode(box, batch_anchors)
    if dir_cls is not None:
        labels = torch.max(dir_cls, dim=-1)[1]
        period = 2 * np.pi / num_dir_bins
        rot = torch_limit_period(out[..., 6] - dir_offset, dir_limit_offset, period)
        out[..., 6] = rot + dir_offset + period * labels.to(out.dtype)
    return out


def torch_rotate_points_along_z(points, angle):
    """common_utils.rotate_points_along_z without the .float() on the matrix (so that float64 stays float64)"""
    cosa, sina = torch.cos(angle), torch.sin(angle)
    zeros, ones = angle.new_zeros(points.shape[0]), angle.new_ones(points.shape[0])
    rot = torch.stack((cosa, sina, zeros, -sina, cosa, zeros, zeros, zeros, ones), dim=1).view(-1, 3, 3)
    return torch.cat((torch.matmul(points[:, :, 0:3], rot), points[:, :, 3:]), dim=-1)


def torch_roi_decode(box, rois):
    """RoIHeadTemplate.generate_predicted_boxes' box branch: box [B * N, 7], rois [B, N, >= 7] -> [B, N, 7]"""
    B = rois.shape[0]
    bp = box.view(B, -1, 7)
    roi_ry = rois[:, :, 6].view(-1)
    roi_xyz = rois[:, :, 0:3].view(-1, 3)
    local_rois = rois.clone()
    local_rois[:, :, 0:3] = 0
    bp = torch_decode(bp, local_rois[..., :7]).view(-1, 7)
    bp = torch_rotate_points_along_z(bp.unsqueeze(dim=1), roi_ry).squeeze(dim=1)
    bp[:, 0:3] += roi_xyz
    return bp.view(B, -1, 7)


def _torch_x(boxes, p, backward):
    """X_TRANS.backward_with_param / forward_with_param on one scene's boxes with p = (rotation, flip, scale)"""
    def rotation(b, sign):
        rot = p[0].unsqueeze(0)
        b[:, 0:3] = torch_rotate_points_along_z(b[None, :, 0:3], sign * rot)[0]
        b[:, 6] += sign * rot
        return b

    def flip(b):
        if p[1]:                            # the reference's host read
            b[:, 1] = -(b[:, 1] + 0)
            b[:, 6] = -(b[:, 6] + 0)
        return b

    if backward:
        boxes[:, 0:6] /= p[2]
        return rotation(flip(boxes), -1)
    boxes = flip(rotation(boxes, 1))
    boxes[:, 0:6] *= p[2]
    return boxes


def _torch_stage_loop(rois, transform_param, frm, to):
    rois = rois.clone()
    out = []
    for b in range(len(rois)):
        cur = rois[b]
        if frm is not None:
            cur = _torch_x(cur, transform_param[b][frm], True)
        if to is not None:
            cur = _torch_x(cur, transform_param[b][to], False)
        out.append(cur)
    return torch.stack(out)


def torch_roi_x_trans(rois, i, transform_param):
    i = clamp_stage(i, len(transform_param[0]))
    return _torch_stage_loop(rois, transform_param, i - 1, i)


def torch_roi_score_trans(rois, i, transform_param):
    i = clamp_stage(i, len(transform_param[0]))
    return _torch_stage_loop(rois, transform_param, i, 0)


def torch_pred_x_trans(preds, i, transform_param):
    i = clamp_stage(i, len(transform_param[0]))
    return _torch_stage_loop(preds, transform_param, i, None)
