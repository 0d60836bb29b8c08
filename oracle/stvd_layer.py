"""numpy restatement of the device-drawn StVD layer discard (csrc/stvd_layer.cu, vc_stvd_layer_keep) — TEST INFRASTRUCTURE.

The reference keeps `np.random.permutation(n)[:int(n * (1 - rate))]` rows (`layer_voxel_discard`, spconv_backbone.py:
134-147).  The device draw keeps a subset of the same size and law, from a counter-based generator:
  * u_i = word 0 of Philox4x32-10(counter (i, site, 0, 0), key (seed & 0xffffffff, seed >> 32));
  * the kept rows are the k = int(n * (1 - rate)) rows with the smallest (u_i, i), in ascending row order.
"""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr [..., 4], key [..., 2] uint32 (broadcast) -> [..., 4] uint32 (Salmon et al., SC'11; 10 rounds)."""
    ctr = np.asarray(ctr, dtype=np.uint64)
    key = np.asarray(key, dtype=np.uint64)
    c0, c1, c2, c3 = (ctr[..., j] for j in range(4))
    k0, k1 = key[..., 0], key[..., 1]
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(W0)) & MASK
            k1 = (k1 + np.uint64(W1)) & MASK
        p0, p1 = M0 * c0, M1 * c2                      # < 2**64: exact in uint64
        hi0, lo0 = p0 >> np.uint64(32), p0 & MASK
        hi1, lo1 = p1 >> np.uint64(32), p1 & MASK
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
    return np.stack(np.broadcast_arrays(c0, c1, c2, c3), -1).astype(np.uint32)


def seed_key(seed):
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return np.array([s & 0xFFFFFFFF, s >> 32], dtype=np.uint32)


def row_keys(n, site, seed):
    """u_i, i < n: word 0 of Philox4x32-10 with counter (i, site, 0, 0)."""
    i = np.arange(n, dtype=np.uint64)
    ctr = np.stack([i, np.full(n, site, np.uint64), np.zeros(n, np.uint64), np.zeros(n, np.uint64)], -1)
    return philox4x32_10(ctr, seed_key(seed))[:, 0]


def keep_count(n, rate):
    return int(n * (1 - rate))


def select(u, k):
    """Rows with the k smallest (u_i, i), ascending."""
    u = np.asarray(u, dtype=np.uint32)
    i = np.arange(u.shape[0])
    return np.sort(np.lexsort((i, u))[:k]).astype(np.int32)


def keep_rows(n, rate, site, seed, keys=None):
    u = row_keys(n, site, seed) if keys is None else np.asarray(keys, dtype=np.uint32)
    return select(u, keep_count(n, rate))
