"""Float64 numpy restatement of the part-score RoI pooling rules R1-R4 of virconv_b200/csrc/part_pool.cu (TEDMHead's
PART branch: gen_sample_grid, bilinear_interpolate_torch_gridsample and the mean of obtain_conf_preds), forward and
closed-form backward.  tests/golden/part_pool_ref.npz, recorded from the reference's own code, checks it."""
from __future__ import annotations

import numpy as np

# tap offsets (dx, dy) in torch's order nw, ne, sw, se
TAPS = ((0, 0), (1, 0), (0, 1), (1, 1))


def positions(rois, S, offsets, scale, H, W, dtype=np.float64):
    """R1 + R2: (ix, iy) [..., S*S] in pixel units of the part map, every operation in `dtype`.  The index grid i / (S - 1)
    is rounded to fp32 in either dtype, as the reference's `.float()` on nonzero()'s indices does (ted_head.py:114)."""
    t = (np.arange(S, dtype=np.float32) / np.float32(S - 1)).astype(dtype)
    i, j = np.divmod(np.arange(S * S), S)
    r = np.asarray(rois).astype(dtype)
    f = lambda v: dtype(v)      # noqa: E731
    dx, dy = r[..., 3:4], r[..., 4:5]
    lx = t[i] * dx - dx / f(2)
    ly = t[j] * dy - dy / f(2)
    c, s = np.cos(r[..., 6:7]), np.sin(r[..., 6:7])
    gx = lx * c + ly * (-s) + f(1) * f(0) + r[..., 0:1]
    gy = lx * s + ly * c + f(1) * f(0) + r[..., 1:2]
    X = (gx + f(offsets[0])) * f(scale)
    Y = (gy + f(offsets[1])) * f(scale)
    ix = ((X / f(W) * f(2) - f(1) + f(1)) * f(W) - f(1)) / f(2)
    iy = ((Y / f(H) * f(2) - f(1) + f(1)) * f(H) - f(1)) / f(2)
    return ix, iy


def taps(ix, iy, H, W):
    """[(x, y, w, inside)] for nw, ne, sw, se: integer coordinates, torch's bilinear weights, the in-bounds mask"""
    x0, y0 = np.floor(ix), np.floor(iy)
    x1, y1 = x0 + 1, y0 + 1
    w = ((x1 - ix) * (y1 - iy), (ix - x0) * (y1 - iy), (x1 - ix) * (iy - y0), (ix - x0) * (iy - y0))
    out = []
    for (ddx, ddy), wk in zip(TAPS, w):
        x, y = x0 + ddx, y0 + ddy
        inside = (x >= 0) & (x <= W - 1) & (y >= 0) & (y <= H - 1)
        out.append((np.where(inside, x, 0).astype(np.int64), np.where(inside, y, 0).astype(np.int64), wk, inside))
    return out


def forward(parts, rois, S, offsets, scale):
    """parts [B, S*S, H, W], rois [B, N, >= 7] -> [B * N, 1] float64 (R1-R3)"""
    parts = np.asarray(parts, np.float64)
    B, S2, H, W = parts.shape
    N = rois.shape[1]
    ix, iy = positions(rois, S, offsets, scale, H, W)
    b = np.arange(B)[:, None, None]
    p = np.arange(S2)[None, None, :]
    v = np.zeros((B, N, S2))
    for x, y, w, inside in taps(ix, iy, H, W):
        v += np.where(inside, parts[b, p, y, x] * w, 0.0)
    return (v.sum(-1) / S2).reshape(B * N, 1)


def backward(rois, g, shape, S, offsets, scale):
    """d out / d parts for the upstream gradient g [B * N] (R4): [B, S*S, H, W] float64"""
    B, S2, H, W = shape
    N = rois.shape[1]
    ix, iy = positions(rois, S, offsets, scale, H, W)
    gs = (np.asarray(g, np.float64).reshape(B, N, 1) / S2) * np.ones((1, 1, S2))
    b = np.broadcast_to(np.arange(B)[:, None, None], (B, N, S2))
    p = np.broadcast_to(np.arange(S2)[None, None, :], (B, N, S2))
    d = np.zeros(shape)
    for x, y, w, inside in taps(ix, iy, H, W):
        np.add.at(d, (b[inside], p[inside], y[inside], x[inside]), (gs * w)[inside])
    return d
