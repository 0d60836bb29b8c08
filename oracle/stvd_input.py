"""numpy restatement of the device-drawn input front end (csrc/stvd.cu, vc_stvd_input_front_end) — TEST INFRASTRUCTURE.

Per scene of the collated cloud [N, W] (rows (b, x, y, z, ..., indicator), scenes contiguous):
  * split: indicator 2 = LiDAR, 1 = virtual (dataset.py:272,284), row order kept;
  * plan: the reference's position / per_bin / out_n arithmetic (dataset.py:120-189, restated by `plan`) from the per-bin
    counts; a scene without virtual points is status 1 (the reference raises ZeroDivisionError);
  * draw: a subsampled bin keeps its `take` smallest (u_i, i), u_i = word 0 of Philox4x32-10 with counter (i, 0, 1, draw),
    i the collated row, in row order (`take` = len(permutation(cnt)[:per_bin]));
  * assembly: [LiDAR, kept bins far -> near] (later_fusion False, intensity / 10) or LiDAR and kept virtual apart;
  * mask_points_by_range (x, y, bounds inclusive), then, when shuffling, each scene's block of each stream permuted by
    `feistel` (counter domain 2).
"""
from __future__ import annotations

import numpy as np

from . import stvd_layer as osl


def bins(x, bin_num, max_dis=60):
    """bin of every point (-1: none), the masks of `DatasetTemplate.partition` (oracle/stvd.py)."""
    inter = max_dis / bin_num
    f32 = np.float32
    b = np.full(x.shape[0], -1, np.int64)
    for i in range(bin_num):
        if i == bin_num - 1:
            m = x >= f32(inter * i)
        else:
            m = (x >= f32(inter * i)) & (x < f32(inter * (i + 1)))
        b[m] = i
    return b


def plan(counts, n_all, bin_num, rate):
    """counts [bin_num] by bin id -> (position, per_bin, out_n, take [bin_num]); take -1 keeps the whole bin.  Raises
    ZeroDivisionError on n_all == 0, as the reference does."""
    retain = 1 - rate
    acc, position, distant_acc = 0, bin_num - 1, 0
    for it in range(bin_num):
        i = bin_num - it - 1
        cnt = int(counts[i])
        acc += cnt
        if (acc + i * cnt) / n_all < retain:
            position = i
            distant_acc = acc
    position = max(position, 0)
    out_n = int(n_all * retain)
    per_bin = int((out_n - distant_acc) / (position + 0.0001))
    take = np.full(bin_num, -1, np.int64)
    for it in range(bin_num):
        i = bin_num - it - 1
        cnt = int(counts[i])
        if it >= bin_num - position and cnt > per_bin:
            take[i] = len(range(cnt)[:per_bin])         # python slice semantics (per_bin < 0)
    return position, per_bin, out_n, take


def feistel(x, n, tweak, draw, seed):
    """The device's bijection of [0, n): a balanced Feistel network of four Philox rounds on 2h bits, cycle-walking."""
    x = np.asarray(x, dtype=np.uint64).copy()
    if n <= 1:
        return x.astype(np.int64)
    bits = int(n - 1).bit_length()
    h = (bits + 1) // 2
    mask = np.uint64((1 << h) - 1)
    key = osl.seed_key(seed)
    todo = np.ones(x.shape[0], bool)
    while todo.any():
        v = x[todo]
        l, r = v >> np.uint64(h), v & mask
        for rd in range(4):
            ctr = np.stack([r, np.full_like(r, tweak), np.full_like(r, 2), np.full_like(r, (draw << 8) | rd)], -1)
            f = osl.philox4x32_10(ctr, key)[:, 0].astype(np.uint64) & mask
            l, r = r, l ^ f
        v = (l << np.uint64(h)) | r
        x[todo] = v
        todo[todo] = v >= np.uint64(n)
    return x.astype(np.int64)


def front_end(points, batch_size, bin_num, rate, later_fusion, shuffle, seed, draw=0,
              pc_range=(0, -40, -3, 70.4, 40, 1), max_dis=60):
    """-> dict(points, src_points, points_mm, src_mm (later_fusion), status [B]): exact-size arrays."""
    pts = np.asarray(points, dtype=np.float32)
    n, w = pts.shape
    rows = np.arange(n)
    b = pts[:, 0]
    ok_b = (b >= 0) & (b < np.float32(batch_size))
    scene = np.where(ok_b, np.where(ok_b, b, 0).astype(np.int64), -1)
    ind = pts[:, -1]
    lo = np.asarray(pc_range, dtype=np.float32)
    in_range = (pts[:, 1] >= lo[0]) & (pts[:, 1] <= lo[3]) & (pts[:, 2] >= lo[1]) & (pts[:, 2] <= lo[4])
    streams = ([], []) if later_fusion else ([],)
    status = np.zeros(batch_size, np.int32)
    for s in range(batch_size):
        lidar = rows[(scene == s) & (ind == 2)]
        virt = rows[(scene == s) & (ind == 1)]
        kept = []
        if virt.shape[0] == 0:
            status[s] = 1
        else:
            vb = bins(pts[virt, 1], bin_num, max_dis)
            counts = np.bincount(vb[vb >= 0], minlength=bin_num)
            _, _, _, take = plan(counts, virt.shape[0], bin_num, rate)
            for i in range(bin_num - 1, -1, -1):
                members = virt[vb == i]
                if take[i] >= 0:
                    u = osl.philox4x32_10(np.stack([members, np.zeros_like(members), np.ones_like(members),
                                                    np.full_like(members, draw)], -1).astype(np.uint64), osl.seed_key(seed))[:, 0]
                    members = members[osl.select(u, int(take[i]))]
                kept.append(members)
        kept = np.concatenate(kept) if kept else np.zeros(0, np.int64)
        blocks = [lidar, kept] if later_fusion else [np.concatenate([lidar, kept])]
        for st, blk in enumerate(blocks):
            blk = blk[in_range[blk]]
            if shuffle:
                perm = feistel(np.arange(blk.shape[0]), blk.shape[0], (st << 16) | s, draw, seed)
                out = np.empty_like(blk)
                out[perm] = blk
                blk = out
            streams[st].append(blk)
    res = {'status': status}
    for st, name in enumerate(('points', 'points_mm')[:len(streams)]):
        src = np.concatenate(streams[st]).astype(np.int64) if streams[st] else np.zeros(0, np.int64)
        out = pts[src].copy()
        if not later_fusion:
            out[:, 4] = out[:, 4] / np.float32(10)
        res[name], res['src_' + name] = out, src
    return res

