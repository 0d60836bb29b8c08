"""Model-side GPU versions of the steps immediately BEFORE the backbone (SURVEY §8f row 1), which the reference runs on the
CPU inside its dataloader workers:

  * `input_point_discard`  — StVD input discard of the virtual points (`DatasetTemplate.partition` +
    `input_point_discard`, pcdet/datasets/dataset.py:120-189), same rows in the same order for the same numpy RNG state;
  * `split_and_discard`    — the per-frame flow around it (dataset.py:270-298): split by the indicator column, discard the
    virtual points, re-fuse (VirConv-L, LATER_FUSION False, intensity / 10) or keep two streams (VirConv-T/S);
  * `PointsToVoxels`       — `DataProcessor.transform_points_to_voxels` (data_processor.py:128-187, spconv's first-come
    `Point2VoxelCPU3d`) fused with `MeanVFE.forward` (mean_vfe.py:39-58): `batch_dict['points']` -> `voxel_features`,
    `voxel_coords`, `voxel_num_points` (and the `_mm` stream), through `vc_voxelize_mean`.

CUDA tensors only; the kernels are in csrc/stvd.cu and csrc/voxelize.cu.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from . import _lib, ops
from ._lib import check


def _discard_plan(counts, n_all, bin_num, rate, rng):
    """Host half of the discard: from the bin sizes alone, the reference's `position` / `per_bin` arithmetic
    (dataset.py:133-166 and :172-178) and the permutations of the subsampled bins (:182-186), drawn from `rng` in the
    order the reference draws them (far -> near over the nearest `position` bins).
    -> (segments [(bin, out_base, count, sel_base)], concatenated selection ranks int32, n_out)."""
    retain = 1 - rate
    acc, position, distant_acc = 0, bin_num - 1, 0
    for it in range(bin_num):                       # far -> near
        i = bin_num - it - 1
        cnt = int(counts[i])
        acc += cnt
        if (acc + i * cnt) / n_all < retain:        # ZeroDivisionError on an empty cloud, like the reference
            position = i
            distant_acc = acc
    position = max(position, 0)
    out_n = int(n_all * retain)
    per_bin = int((out_n - distant_acc) / (position + 0.0001))
    segs, sels, out_base, sel_base = [], [], 0, 0
    for it in range(bin_num):
        i = bin_num - it - 1
        cnt = int(counts[i])
        if it >= bin_num - position and cnt > per_bin:
            sel = np.asarray(rng.permutation(cnt)[:per_bin], dtype=np.int32)     # python slice semantics kept (per_bin < 0)
            segs.append((i, out_base, len(sel), sel_base if len(sel) else -1))    # an emptied bin needs no list
            sels.append(sel)
            sel_base += len(sel)
            out_base += len(sel)
        else:
            segs.append((i, out_base, cnt, -1))
            out_base += cnt
    sel_all = np.concatenate(sels) if sels else np.zeros(0, dtype=np.int32)
    return segs, sel_all, out_base


def input_point_discard(points, bin_num=2, rate=0.8, rng=None, max_dis=60):
    """Bin-based StVD discard of one sample's points [N, C] fp32 CUDA (x in column 0) -> [M, C], rows and order identical
    to the reference's numpy version for the same generator state (`rng` defaults to the global `np.random`, which is what
    the reference draws from).  One host read (the <= 16 bin sizes), two kernel sequences."""
    ops._require_cuda(points)
    lib = _lib.load()
    assert points.dim() == 2 and points.dtype == torch.float32
    points = points.contiguous()
    rng = np.random if rng is None else rng
    n, c = points.shape
    if n == 0:
        raise ZeroDivisionError('input_point_discard on an empty point cloud (the reference divides by the point count)')
    dev = points.device
    totals = torch.empty(16, dtype=torch.int32, device=dev)
    ws = ops._ws(lib.vc_stvd_ws_bytes(n), dev)
    check(lib.vc_stvd_partition(points.data_ptr(), n, c, int(bin_num), float(max_dis), totals.data_ptr(), ws.data_ptr(),
                                ws.numel(), ops._stream()), 'vc_stvd_partition')
    counts = totals.cpu().numpy()                   # the one host read: bin sizes
    segs, sel, n_out = _discard_plan(counts, n, int(bin_num), rate, rng)
    out = torch.empty((n_out, c), dtype=torch.float32, device=dev)
    sel_dev = torch.from_numpy(sel).to(dev) if len(sel) else None
    flat = [v for s in segs for v in s]
    check(lib.vc_stvd_gather(points.data_ptr(), n, c, _lib.host_i32(flat), len(segs),
                             sel_dev.data_ptr() if sel_dev is not None else None, out.data_ptr(), n_out, ws.data_ptr(),
                             ws.numel(), ops._stream()), 'vc_stvd_gather')
    return out


def split_and_discard(points, training, input_discard_rate=0.8, later_fusion=False, rng=None):
    """One frame's `points` [N, C] (last column = indicator: 1 virtual, 2 LiDAR) -> dict, as dataset.py:270-298:
    virtual points go through the StVD discard (bin_num 2 when training, 10 at test time); VirConv-L (`later_fusion`
    False) re-fuses `[lidar, kept virtual]` and divides the intensity column by 10, VirConv-T/S keep `points` (LiDAR) and
    `points_mm` (virtual) apart."""
    ops._require_cuda(points)
    ind = points[:, -1]
    virt = points[ind == 1]
    lidar = points[ind == 2]
    kept = input_point_discard(virt, bin_num=2 if training else 10, rate=input_discard_rate, rng=rng)
    if later_fusion:
        return {'points': lidar, 'points_mm': kept}
    fused = torch.cat([lidar, kept])
    # IEEE division like numpy's `points[:, 3] /= 10` (:294); torch's tensor / python-scalar on CUDA multiplies by the
    # rounded reciprocal instead, which is 1 ulp off for some values
    fused[:, 3] = torch.div(fused[:, 3], torch.full((), 10.0, dtype=torch.float32, device=fused.device))
    return {'points': fused}


_I64 = torch.iinfo(torch.int64)


def input_front_end(points, batch_size, training, later_fusion, rate=0.8, seed=None, n_dev=None,
                    point_cloud_range=(0, -40, -3, 70.4, 40, 1), bin_num=None, shuffle=None, draw=0, cap=None, static=False,
                    max_dis=60, overflow=None):
    """The dataloader's per-frame input flow for a whole collated batch, with every draw on the device and no host read
    (vc_stvd_input_front_end, csrc/stvd.cu): `points` [N, 1+C] fp32 (b, x, y, z, ..., indicator), scenes contiguous, as
    `collate_batch` builds it before any split; n_dev (device int32[1]) its valid rows when it is a capacity-sized buffer.

    Per scene: split by the indicator (dataset.py:272,284), the StVD input discard of the virtual points (bin_num 2 when
    training, 10 at test time; keys from Philox under `seed`, a device int64[1], default one fresh draw of torch's CUDA
    generator), [LiDAR, kept virtual] with intensity / 10 (later_fusion False, VirConv-L) or the two streams apart
    (VirConv-T / -S), mask_points_by_range, and when shuffling (default: training) a per-scene pseudo-random permutation of every
    stream, as the reference's shuffle_points does for 'points' and, with two streams, 'points_mm' (data_processor.py:
    105-124).  `draw` separates independent draws under one seed (the ROT_NUM copies).

    -> {'points', 'points_mm' (later_fusion), 'stvd_input_kept' (the input row of every 'points' row, and with two streams
    'stvd_input_kept_mm'), 'stvd_input_status' [B] int32 (1: a scene without virtual points, where the reference raises
    ZeroDivisionError), 'stvd_input_overflow' int32[1]}.  static=False: exact-size tensors (one host read of the two row
    counts).  static=True: capacity-sized ones (cap rows, default the input's), tail rows (-1, 0, ...) that the voxeliser
    drops, each stream tensor carrying its device row count as `.num_rows`; the overflow word (`overflow`, a device int32[1]
    the call raises to the rows that did not fit, or a fresh zero one) holds the rows that did not fit, and also the rows
    dropped because the scenes were not contiguous and ascending."""
    ops._require_cuda(points, n_dev, seed)
    lib = _lib.load()
    assert points.dim() == 2 and points.dtype == torch.float32, (points.dtype, points.shape)
    points = points.contiguous()
    n, w = points.shape
    dev = points.device
    bin_num = int(bin_num if bin_num is not None else (2 if training else 10))
    shuffle = bool(training if shuffle is None else shuffle)
    if seed is None:
        seed = torch.randint(_I64.min, _I64.max, (1,), dtype=torch.int64, device=dev)
    assert seed.dtype == torch.int64 and seed.numel() == 1 and seed.device == dev
    if n_dev is not None:
        assert n_dev.dtype == torch.int32 and n_dev.numel() == 1
    cap = n if cap is None else int(cap)
    names = ('points', 'points_mm') if later_fusion else ('points',)
    outs = [torch.empty((cap, w), dtype=torch.float32, device=dev) for _ in names]
    srcs = [torch.empty((cap,), dtype=torch.int32, device=dev) for _ in names]
    counts = torch.empty(2, dtype=torch.int32, device=dev)
    status = torch.empty(int(batch_size), dtype=torch.int32, device=dev)
    if overflow is None:
        overflow = torch.zeros(1, dtype=torch.int32, device=dev)
    assert overflow.dtype == torch.int32 and overflow.numel() == 1 and overflow.device == dev
    ws = ops._ws(lib.vc_stvd_input_ws_bytes(n, int(batch_size)), dev)
    mm = later_fusion
    check(lib.vc_stvd_input_front_end(points.data_ptr(), n, ops._p(n_dev), w, int(batch_size), bin_num, float(max_dis), float(rate),
                                      _lib.host_f32(point_cloud_range), int(bool(later_fusion)), int(shuffle), seed.data_ptr(),
                                      int(draw), outs[0].data_ptr(), srcs[0].data_ptr(), cap,
                                      outs[1].data_ptr() if mm else None, srcs[1].data_ptr() if mm else None, cap if mm else 0,
                                      counts.data_ptr(), status.data_ptr(), overflow.data_ptr(), ws.data_ptr(), ws.numel(),
                                      ops._stream()), 'vc_stvd_input_front_end')
    res = {'stvd_input_status': status, 'stvd_input_overflow': overflow}
    rows = counts.tolist() if not static else None
    for i, (name, o, s) in enumerate(zip(names, outs, srcs)):
        if static:
            o.num_rows = s.num_rows = counts[i:i + 1]
        else:
            o, s = o[:rows[i]], s[:rows[i]]
        res[name] = o
        res['stvd_input_kept' + name[len('points'):]] = s
    return res


class PointsToVoxels(nn.Module):
    """Voxelisation + VFE as a model-side module: reads `batch_dict['points']` ([N, 1+C] fp32 rows (b, x, y, z, ...),
    samples contiguous in batch order — what `collate_batch` builds, dataset.py:349-353) and writes what the dataloader's
    `transform_points_to_voxels` + `MeanVFE` would have: `voxel_features` [M, C], `voxel_coords` [M, 4] (b, z, y, x),
    `voxel_num_points` [M]; likewise `points_mm` -> `*_mm`.  Same first-come voxel order, same per-voxel point cap."""

    def __init__(self, voxel_size=(0.05, 0.05, 0.05), point_cloud_range=(0, -40, -3, 70.4, 40, 1), max_points_per_voxel=5,
                 max_voxels=40000, vfe_model='max', float_coords=True):
        super().__init__()
        self.voxel_size, self.point_cloud_range = tuple(voxel_size), tuple(point_cloud_range)
        self.max_points_per_voxel, self.max_voxels, self.vfe_model = int(max_points_per_voxel), max_voxels, vfe_model
        self.float_coords = float_coords          # `load_data_to_gpu` ships coordinates as float32 (models/__init__.py:16-24)

    def _max_voxels(self):
        mv = self.max_voxels
        if isinstance(mv, dict):                  # MAX_NUMBER_OF_VOXELS: {train, test} (data_processor.py:144)
            mv = mv['train' if self.training else 'test']
        return int(mv)

    def forward(self, batch_dict):
        bs = int(batch_dict['batch_size'])
        for sfx in ('', '_mm'):
            key = 'points' + sfx
            if key not in batch_dict:
                continue
            f, c, n = ops.voxelize_mean(batch_dict[key], bs, self.point_cloud_range, self.voxel_size,
                                        self.max_points_per_voxel, self._max_voxels(), self.vfe_model)
            batch_dict['voxel_features' + sfx] = f
            batch_dict['voxel_coords' + sfx] = c.float() if self.float_coords else c
            batch_dict['voxel_num_points' + sfx] = n
        return batch_dict
