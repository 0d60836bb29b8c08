"""float64 restatement of the rotated-box IoU / NMS rules that virconv_b200/csrc/iou3d_nms.cu states (rules 1-5 of its
header; the reference's pcdet/ops/iou3d_nms).  TEST INFRASTRUCTURE (see oracle/__init__.py).

Written from the rules, per pair in plain Python floats; matrices skip pairs whose bounds (padded past the 1 cm margin)
are disjoint, whose vertex set is empty."""
from __future__ import annotations

import math

import numpy as np

MARGIN = 0.01
PAD = 0.02


def corners(box):
    """rule 1: the 4 corners of the BEV rectangle, counter-clockwise from (-dx/2, -dy/2)"""
    x, y, _, dx, dy, _, h = (float(v) for v in box[:7])
    c, s = math.cos(h), math.sin(h)
    return [(x + lx * c - ly * s, y + lx * s + ly * c)
            for lx, ly in ((-dx / 2, -dy / 2), (dx / 2, -dy / 2), (dx / 2, dy / 2), (-dx / 2, dy / 2))]


def _cross(p1, p2, p0):
    return (p1[0] - p0[0]) * (p2[1] - p0[1]) - (p2[0] - p0[0]) * (p1[1] - p0[1])


def _crossing(p0, p1, q0, q1):
    """rule 2a: crossing point of segment p0-p1 with q0-q1, or None"""
    if not (min(p0[0], p1[0]) <= max(q0[0], q1[0]) and min(q0[0], q1[0]) <= max(p0[0], p1[0])
            and min(p0[1], p1[1]) <= max(q0[1], q1[1]) and min(q0[1], q1[1]) <= max(p0[1], p1[1])):
        return None
    s1, s2 = _cross(q0, p1, p0), _cross(p1, q1, p0)
    s3, s4 = _cross(p0, q1, q0), _cross(q1, p1, q0)
    if not (s1 * s2 > 0 and s3 * s4 > 0):
        return None
    s5 = _cross(q1, p1, p0)
    if abs(s5 - s1) > 1e-8:
        return ((s5 * q0[0] - s1 * q1[0]) / (s5 - s1), (s5 * q0[1] - s1 * q1[1]) / (s5 - s1))
    a0, b0, c0 = p0[1] - p1[1], p1[0] - p0[0], p0[0] * p1[1] - p1[0] * p0[1]
    a1, b1, c1 = q0[1] - q1[1], q1[0] - q0[0], q0[0] * q1[1] - q1[0] * q0[1]
    d = a0 * b1 - a1 * b0
    return ((b0 * c1 - b1 * c0) / d, (a1 * c0 - a0 * c1) / d)


def _inside(box, p):
    """rule 2b: p inside the box with the 1 cm margin"""
    x, y, _, dx, dy, _, h = (float(v) for v in box[:7])
    c, s = math.cos(h), math.sin(h)
    lx = (p[0] - x) * c + (p[1] - y) * s
    ly = -(p[0] - x) * s + (p[1] - y) * c
    return abs(lx) < dx / 2 + MARGIN and abs(ly) < dy / 2 + MARGIN


def overlap(a, b):
    """rules 2-3: BEV intersection area"""
    ca, cb = corners(a), corners(b)
    pts = []
    for i in range(4):
        for j in range(4):
            p = _crossing(ca[i], ca[(i + 1) % 4], cb[j], cb[(j + 1) % 4])
            if p is not None:
                pts.append(p)
    for k in range(4):
        if _inside(a, cb[k]):
            pts.append(cb[k])
        if _inside(b, ca[k]):
            pts.append(ca[k])
    if len(pts) < 3:
        return 0.0
    mx = sum(p[0] for p in pts) / len(pts)
    my = sum(p[1] for p in pts) / len(pts)
    pts = sorted(pts, key=lambda p: math.atan2(p[1] - my, p[0] - mx))      # sorted() is stable
    v0 = pts[0]
    area = sum((pts[k][0] - v0[0]) * (pts[k + 1][1] - v0[1]) - (pts[k][1] - v0[1]) * (pts[k + 1][0] - v0[0])
               for k in range(len(pts) - 1))
    return abs(area) / 2


def iou_bev(a, b):
    ov = overlap(a, b)
    return ov / max(float(a[3]) * float(a[4]) + float(b[3]) * float(b[4]) - ov, 1e-8)


def iou3d(a, b):
    ov = overlap(a, b)
    h = max(min(float(a[2]) + float(a[5]) / 2, float(b[2]) + float(b[5]) / 2)
            - max(float(a[2]) - float(a[5]) / 2, float(b[2]) - float(b[5]) / 2), 0.0)
    o3 = ov * h
    va = float(a[3]) * float(a[4]) * float(a[5])
    vb = float(b[3]) * float(b[4]) * float(b[5])
    return o3 / max(va + vb - o3, 1e-6)


def iou_normal(a, b):
    """rule 4: axis-aligned IoU, heading ignored"""
    ax, ay, adx, ady = (float(a[i]) for i in (0, 1, 3, 4))
    bx, by, bdx, bdy = (float(b[i]) for i in (0, 1, 3, 4))
    w = max(min(ax + adx / 2, bx + bdx / 2) - max(ax - adx / 2, bx - bdx / 2), 0.0)
    h = max(min(ay + ady / 2, by + bdy / 2) - max(ay - ady / 2, by - bdy / 2), 0.0)
    inter = w * h
    return inter / max(adx * ady + bdx * bdy - inter, 1e-8)


def _bounds(boxes):
    b = np.asarray(boxes, np.float64)
    c, s = np.abs(np.cos(b[:, 6])), np.abs(np.sin(b[:, 6]))
    ex = (b[:, 3] * c + b[:, 4] * s) / 2 + PAD
    ey = (b[:, 3] * s + b[:, 4] * c) / 2 + PAD
    return b[:, 0] - ex, b[:, 0] + ex, b[:, 1] - ey, b[:, 1] + ey


def matrix(boxes_a, boxes_b, fn=iou_bev):
    """[Na, Nb] float64 of fn over every pair; pairs with disjoint padded bounds are 0 (their vertex set is empty)"""
    A, B = np.asarray(boxes_a, np.float64), np.asarray(boxes_b, np.float64)
    out = np.zeros((len(A), len(B)))
    if fn is iou_normal:
        cand = np.ones((len(A), len(B)), bool)
    else:
        al, ah, ad, au = _bounds(A)
        bl, bh, bd, bu = _bounds(B)
        cand = (al[:, None] <= bh[None]) & (bl[None] <= ah[:, None]) & (ad[:, None] <= bu[None]) & (bd[None] <= au[:, None])
    for i, j in zip(*np.nonzero(cand)):
        out[i, j] = fn(A[i], B[j])
    return out


def nms(boxes_sorted, thresh, normal=False):
    """rule 5: greedy over boxes already sorted by descending score -> kept row indices"""
    B = np.asarray(boxes_sorted, np.float64)
    iou = matrix(B, B, iou_normal if normal else iou_bev)
    removed = np.zeros(len(B), bool)
    keep = []
    for i in range(len(B)):
        if removed[i]:
            continue
        keep.append(i)
        removed[i + 1:] |= iou[i, i + 1:] > thresh
    return np.array(keep, np.int64)
