"""Numpy restatement of the test-time x-batching of VirConv8x (csrc/xbatch.cu).  TEST INFRASTRUCTURE (see oracle/__init__.py).

The reference's eval forward (`pcdet/models/backbones_3d/spconv_backbone.py:408-471`) shifts transformed copy i of the LiDAR
voxels by i*W along x, concatenates the copies into one [D, H, 4W] tensor (:418-432; the factor 4 is fixed at :360) and
splits the published tensors back with `decompose_tensor` (:314-337): copy i keeps the rows with i*q < x < (i+1)*q,
q = W' // 4 — strict on both sides, the x == i*q column belongs to no copy — and moves them back by i*q.  Both functions
below work on capacity-sized arrays with a valid row count, the static (graph) form of those tensors.
"""
from __future__ import annotations

import numpy as np

MAX_COPIES = 4


def pack(feats, coords, counts, width):
    """Copies (features [cap_i, C], coordinates [cap_i, 4] (b, z, y, x), valid row counts) -> (features [sum cap_i, C],
    coordinates [sum cap_i, 4], total): the valid rows of copy 0, copy 1, ... with x += i * width, zero / -1 tail."""
    assert 1 <= len(feats) <= MAX_COPIES
    cap = sum(f.shape[0] for f in feats)
    c = feats[0].shape[1]
    out_f = np.zeros((cap, c), dtype=np.float32)
    out_c = np.full((cap, 4), -1, dtype=np.int32)
    r = 0
    for i, (f, co, n) in enumerate(zip(feats, coords, counts)):
        n = int(min(max(n, 0), f.shape[0]))
        out_f[r:r + n] = f[:n]
        out_c[r:r + n] = co[:n]
        out_c[r:r + n, 3] += i * width
        r += n
    return out_f, out_c, r


def split(feats, indices, n, width, copies):
    """A tensor of x extent `width` (capacity-sized, `n` valid rows) -> `copies` tuples (features, indices, count), each of
    the parent's capacity: the rows of copy i in order, x -= i*q, zero / -1 tail."""
    assert 1 <= copies <= MAX_COPIES
    cap = feats.shape[0]
    n = int(min(max(n, 0), cap))
    q = width // 4
    x = indices[:n, 3].astype(np.int64)
    out = []
    for i in range(copies):
        rows = np.nonzero((x > i * q) & (x < (i + 1) * q))[0]
        f = np.zeros_like(feats)
        idx = np.full((cap, 4), -1, dtype=np.int32)
        f[:rows.size] = feats[rows]
        idx[:rows.size] = indices[rows]
        idx[:rows.size, 3] -= i * q
        out.append((f, idx, int(rows.size)))
    return out
