"""The front end of TEDMHead's voxel-RoI grid pooling (VirConv-L / -T / -S) on the sm_90a kernel of csrc/roi_grid.cu,
which states the rules.

  * `roi_grid_points`  = get_global_grid_points_of_roi and the voxel coordinates of the grid points (ted_head.py:474-485,
                         :528-532) for all scenes and all feature sources in one launch;
  * `voxel_centers`    = common_utils.get_voxel_centers (common_utils.py:65-81) from the device tensors alone;
  * `roi_grid_pool`, `roi_grid_pool_mm` = the drop-in methods (bound by reference_env.install(use_fused_roi_grid=True)).

The reference reads the device once per call (`nonzero()` in get_dense_grid_points), copies voxel_size and
point_cloud_range from the host twice per source, loops over the scenes in Python and rebuilds the dense voxel -> row map
(generate_voxel2pinds) for every source of every stage and branch, although it depends only on the published tensor.
Here nothing reads the device (the call can be captured in a CUDA graph), and the map and the voxel centres of each
published tensor are built once per batch_dict and shared by every stage and both branches of that forward.

Static-form tensors (capacity-sized, -1 index tail, device row count `.num_rows`, as GraphedForward publishes them) are
accepted: the map is built from the valid rows only, so the tail rows are never pooled.  In training mode the pool
layer's input BatchNorm1d would also normalise over the tail rows, so a static-form tensor is refused there.

Fallbacks to the reference method: a pool layer that is not the fused virconv_b200.voxel_pool.NeighborVoxelSAModuleMSG,
RoIs that require a gradient (the reference lets it flow through grouped_xyz - new_xyz; the fused layer takes none), and
a feature source other than x_conv1..4."""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, ops
from ._lib import check, host_f32, host_i32
from .voxel_pool import NeighborVoxelSAModuleMSG

MAX_SOURCES = 4     # VC_ROI_GRID_MAX_SOURCES
MAX_GRID = 64
SOURCES = ('x_conv1', 'x_conv2', 'x_conv3', 'x_conv4')
CACHE_KEY = '_virconv_b200_roi_grid'    # batch_dict key of the per-forward map / centre cache

_reference_roi_grid_pool = None         # TEDMHead's own methods (set by reference_env)
_reference_roi_grid_pool_mm = None


def _f32(v):
    """v as the float32 value torch's wrapped-scalar rule gives a float32 tensor op, as a Python float"""
    return float(np.float32(v))


def roi_grid_points(rois, grid_size, point_cloud_range, voxel_size, strides):
    """rois [B, N, >= 7] (x, y, z, dx, dy, dz, heading) CUDA fp32, grid size G, point_cloud_range[0:3], voxel_size (3),
    strides (<= 4 source strides) -> new_xyz [B * N * G^3, 3] fp32 (the reference's roi_grid_xyz.view(-1, 3)) and
    new_coords [len(strides), B * N * G^3, 4] int32, (b, x, y, z): the reference's cur_roi_grid_coords of each source.
    One launch; no host read."""
    ops._require_cuda(rois)
    G, S = int(grid_size), len(strides)
    if rois.dtype != torch.float32 or rois.dim() != 3 or rois.shape[2] < 7:
        raise ValueError(f'roi_grid_points: rois must be [B, N, >= 7] float32 (got {tuple(rois.shape)} {rois.dtype})')
    if not 1 <= G <= MAX_GRID or S > MAX_SOURCES:
        raise ValueError(f'roi_grid_points: grid size {G} (1..{MAX_GRID}) with {S} sources (at most {MAX_SOURCES})')
    r = rois.contiguous()
    B, N, ld = r.shape
    M = B * N * G ** 3
    new_xyz = torch.empty((M, 3), dtype=torch.float32, device=r.device)
    new_coords = torch.empty((S, M, 4), dtype=torch.int32, device=r.device)
    check(_lib.load().vc_roi_grid_points(r.data_ptr(), B, N, ld, G, host_f32([_f32(v) for v in point_cloud_range[0:3]]),
                                         host_f32([_f32(v) for v in voxel_size]), host_i32(strides), S, new_xyz.data_ptr(),
                                         new_coords.data_ptr(), ops._stream()), 'vc_roi_grid_points')
    return new_xyz, new_coords


def voxel_centers(indices, stride, voxel_size, point_cloud_range):
    """indices [n, 4] (b, z, y, x) on the device -> [n, 3] fp32 centres (x, y, z): get_voxel_centers(indices[:, 1:4],
    stride, voxel_size, point_cloud_range), the same float32 operations with the constants as float32-exact scalars
    instead of host-built tensors (rows of a -1 tail get meaningless centres no map row points to)."""
    cols = indices[:, 1:4].flip(1).float()
    out = []
    for a in range(3):
        size = _f32(np.float32(voxel_size[a]) * np.float32(stride))       # torch.tensor(voxel_size).float() * stride
        out.append((cols[:, a] + 0.5) * size + _f32(point_cloud_range[a]))
    return torch.stack(out, 1)


def _source(batch_dict, sp, stride, voxel_size, point_cloud_range):
    """(centres, voxel -> row map) of the published tensor `sp`, built once per batch_dict.  The entry keeps `sp` and its
    indices alive, so an identity match cannot come from a recycled id; a static-form tensor refilled for another scene
    comes with a new batch_dict and so with a new cache."""
    cache = batch_dict.get(CACHE_KEY)
    if cache is None:
        cache = batch_dict[CACHE_KEY] = {}
    key = (id(sp), int(stride))
    hit = cache.get(key)
    if hit is not None and hit[0] is sp and hit[1] is sp.indices:
        return hit[2], hit[3]
    idx = sp.indices
    v2p = ops.voxel2pinds(idx, sp.batch_size, sp.spatial_shape, num_rows=getattr(sp, 'num_rows', None))
    xyz = voxel_centers(idx, stride, voxel_size, point_cloud_range)
    cache[key] = (sp, idx, xyz, v2p)
    return xyz, v2p


def _lidar_features(batch_dict, i):
    """the feature dict roi_grid_pool reads (ted_head.py:464-512): rot_num_id with the `while ... not in batch_dict`
    fall-back to lower ids, then multi_scale_3d_features_post when with_voxel_feature_transform"""
    rot_num_id = '' if i == 0 else str(i)
    j = i
    while 'multi_scale_3d_features' + rot_num_id not in batch_dict:
        j -= 1
        if j < 0:       # the reference's loop would count down forever here
            raise KeyError(f'roi_grid_pool: no multi_scale_3d_features{"" if i == 0 else i} in batch_dict and none of a '
                           f'lower stage to fall back to')
        rot_num_id = str(j)
    if batch_dict.get('with_voxel_feature_transform', False):
        return batch_dict['multi_scale_3d_features_post']
    return batch_dict['multi_scale_3d_features' + rot_num_id]


def _mm_features(batch_dict, i):
    """the feature dict roi_grid_pool_mm reads (ted_head.py:567-611): the MM branch's own tensors where published, else
    the LiDAR ones of the same stage"""
    rot_num_id = '' if i == 0 else str(i)
    if batch_dict.get('with_voxel_feature_transform', False):
        return batch_dict['multi_scale_3d_features_post']
    if 'multi_scale_3d_features_mm' + rot_num_id in batch_dict:
        return batch_dict['multi_scale_3d_features_mm' + rot_num_id]
    return batch_dict['multi_scale_3d_features' + rot_num_id]


def _fused_ok(batch_dict, cfg, layers):
    return (not batch_dict['rois'].requires_grad and all(s in SOURCES for s in cfg.FEATURES_SOURCE)
            and all(isinstance(layers[k], NeighborVoxelSAModuleMSG) for k in range(len(cfg.FEATURES_SOURCE))))


def _pool(self, batch_dict, cfg, layers, feats):
    G = int(cfg.GRID_SIZE)
    names = list(cfg.FEATURES_SOURCE)
    strides = [int(batch_dict['multi_scale_3d_strides'][s]) for s in names]
    new_xyz, new_coords = roi_grid_points(batch_dict['rois'], G, self.point_cloud_range, self.voxel_size, strides)
    pooled_list = []
    for k, src in enumerate(names):
        sp = feats[src]
        pool_layer = layers[k]
        if getattr(sp, 'num_rows', None) is not None and pool_layer.training:
            raise ValueError(f'roi_grid_pool: {src} is a static-form tensor (capacity-sized, .num_rows) and the pool layer '
                             f'is in training mode, whose input BatchNorm1d would normalise over the tail rows too; pass '
                             f'exact-size tensors for training')
        xyz, v2p = _source(batch_dict, sp, strides[k], self.voxel_size, self.point_cloud_range)
        pooled = pool_layer(xyz=xyz, xyz_batch_cnt=None, new_xyz=new_xyz, new_xyz_batch_cnt=None,
                            new_coords=new_coords[k], features=sp.features.contiguous(), voxel2point_indices=v2p)
        pooled_list.append(pooled.view(-1, G ** 3, pooled.shape[-1]))
    return torch.cat(pooled_list, dim=-1)


def roi_grid_pool(self, batch_dict, i):
    """TEDMHead.roi_grid_pool (ted_head.py:450-552; bound by reference_env.install(use_fused_roi_grid=True)): the pooled
    features [B * N, G^3, sum C] of stage i's RoIs (batch_dict['rois'] [B, N, >= 7]) over the sources of
    self.pool_cfg, through self.roi_grid_pool_layers.  The batch counts are passed as None: the fused layer reads the
    batch index of new_coords and the global rows of the map instead."""
    if not _fused_ok(batch_dict, self.pool_cfg, self.roi_grid_pool_layers):
        if _reference_roi_grid_pool is None:
            raise RuntimeError('roi_grid_pool: this head needs the reference method, which '
                               'reference_env.install(use_fused_roi_grid=True) records before binding this one')
        return _reference_roi_grid_pool(self, batch_dict, i)
    return _pool(self, batch_dict, self.pool_cfg, self.roi_grid_pool_layers, _lidar_features(batch_dict, i))


def roi_grid_pool_mm(self, batch_dict, i):
    """TEDMHead.roi_grid_pool_mm (ted_head.py:553-650; bound by reference_env.install(use_fused_roi_grid=True)): as
    roi_grid_pool over self.pool_cfg_mm and self.roi_grid_pool_layers_mm, reading the MM branch's tensors and falling back
    to the LiDAR ones of the stage where those are not published."""
    if not _fused_ok(batch_dict, self.pool_cfg_mm, self.roi_grid_pool_layers_mm):
        if _reference_roi_grid_pool_mm is None:
            raise RuntimeError('roi_grid_pool_mm: this head needs the reference method, which '
                               'reference_env.install(use_fused_roi_grid=True) records before binding this one')
        return _reference_roi_grid_pool_mm(self, batch_dict, i)
    return _pool(self, batch_dict, self.pool_cfg_mm, self.roi_grid_pool_layers_mm, _mm_features(batch_dict, i))
