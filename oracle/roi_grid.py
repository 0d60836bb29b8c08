"""Restatements of the front end of TEDMHead's voxel-RoI grid pooling (ted_head.py:450-673), for the tests and the
profile:

  * float32 numpy, rule by rule of csrc/roi_grid.cu: `grid_points` (G1-G3), `div_floor` (torch's div_floor_floating),
    `coords` (G4), `voxel_centers` (common_utils.get_voxel_centers) and `voxel2pinds` (spconv_utils.generate_voxel2pinds);
  * torch, on any device: `reference_roi_grid_pool`, the reference method's control flow as it runs — the grid from
    `nonzero()` (a device-to-host read), the rotation as a batched matmul, host-built constant tensors, per-scene loops
    for the batch index and counts, and a fresh map per source — calling the head's own pool layers.
"""
from __future__ import annotations

import numpy as np

SOURCES = ('x_conv1', 'x_conv2', 'x_conv3', 'x_conv4')
f32 = np.float32


def div_floor(a, b):
    """torch's float floor division (c10/util/generic_math.h div_floor_floating), elementwise in the dtype of a"""
    a = np.asarray(a)
    dt = a.dtype.type
    b = np.broadcast_to(np.asarray(b, a.dtype), a.shape)
    with np.errstate(divide='ignore', invalid='ignore'):
        mod = np.fmod(a, b)
        div = (a - mod) / b
        div = np.where((mod != 0) & ((b < 0) != (mod < 0)), div - dt(1), div)
        fl = np.floor(div)
        fl = np.where(div - fl > dt(0.5), fl + dt(1), fl)
        fl = np.where(div != 0, fl, np.copysign(dt(0), a / b))
        return np.where(b == 0, a / b, fl).astype(a.dtype)


def local_points(rois, G):
    """rois [R, >= 7] -> [R, G^3, 3] float32: get_dense_grid_points (G1, G2)"""
    r = np.asarray(rois, f32).reshape(-1, rois.shape[-1])
    idx = np.stack(np.nonzero(np.ones((G, G, G))), 1).astype(f32)            # x slowest, z fastest
    size = r[:, None, 3:6]
    return ((idx[None] + f32(0.5)) / f32(G)) * size - size / f32(2)


def grid_points(rois, G):
    """rois [B, N, >= 7] -> [B * N * G^3, 3] float32: get_global_grid_points_of_roi (G1-G3)"""
    r = np.asarray(rois, f32).reshape(-1, rois.shape[-1])
    loc = local_points(r, G)
    c, s = np.cos(r[:, 6])[:, None], np.sin(r[:, 6])[:, None]
    zero = f32(0)
    x = (loc[..., 0] * c + loc[..., 1] * -s) + loc[..., 2] * zero
    y = (loc[..., 0] * s + loc[..., 1] * c) + loc[..., 2] * zero
    z = (loc[..., 0] * zero + loc[..., 1] * zero) + loc[..., 2] * f32(1)
    g = np.stack([x, y, z], -1) + r[:, None, 0:3]
    return g.reshape(-1, 3).astype(f32)


def coords(xyz, B, point_cloud_range, voxel_size, stride):
    """grid points [B * P, 3] float32 (scene-major) -> [B * P, 4] int32 (b, x, y, z): (xyz - range) // voxel_size
    // stride, then .int() (G4); the constants as float32, as torch's wrapped-scalar rule rounds them"""
    xyz = np.asarray(xyz, f32)
    v = div_floor(xyz - np.asarray([f32(x) for x in point_cloud_range[0:3]], f32),
                  np.asarray([f32(x) for x in voxel_size], f32))
    v = div_floor(v, f32(stride))
    b = np.repeat(np.arange(B, dtype=np.int32), xyz.shape[0] // B)
    return np.concatenate([b[:, None], np.trunc(v).astype(np.int32)], 1)


def voxel_centers(indices, stride, voxel_size, point_cloud_range):
    """indices [n, 4] (b, z, y, x) -> [n, 3] float32 (x, y, z): get_voxel_centers"""
    c = np.asarray(indices)[:, [3, 2, 1]].astype(f32)
    size = np.asarray([f32(x) for x in voxel_size], f32) * f32(stride)
    return (c + f32(0.5)) * size + np.asarray([f32(x) for x in point_cloud_range[0:3]], f32)


def voxel2pinds(indices, batch_size, spatial_shape, num_rows=None):
    """indices [n, 4] -> [batch_size, *spatial_shape] int32: the row of each voxel, -1 where there is none (rows from
    num_rows on are a static-form tail and are skipped)"""
    idx = np.asarray(indices, np.int64)[:num_rows]
    out = np.full((batch_size, *spatial_shape), -1, np.int32)
    out[tuple(idx.T)] = np.arange(idx.shape[0], dtype=np.int32)
    return out


# ---- the reference method's control flow over torch ----------------------------------------------------------------
def _ref_grid_points(rois, G):
    import torch
    rois = rois.view(-1, rois.shape[-1])
    R = rois.shape[0]
    dense_idx = rois.new_ones((G, G, G)).nonzero().repeat(R, 1, 1).float()
    size = rois.view(R, -1)[:, 3:6]
    local = (dense_idx + 0.5) / G * size.unsqueeze(dim=1) - (size.unsqueeze(dim=1) / 2)
    angle = rois[:, 6]
    cosa, sina = torch.cos(angle), torch.sin(angle)
    zeros, ones = angle.new_zeros(R), angle.new_ones(R)
    rot = torch.stack((cosa, sina, zeros, -sina, cosa, zeros, zeros, zeros, ones), dim=1).view(-1, 3, 3).float()
    return torch.matmul(local[:, :, 0:3], rot) + rois[:, 0:3].unsqueeze(dim=1)


def reference_roi_grid_pool(head, batch_dict, i, mm=False):
    """TEDMHead.roi_grid_pool (mm=False) / roi_grid_pool_mm (mm=True) as the reference runs it, on the head's own pool
    layers"""
    import torch
    cfg = head.pool_cfg_mm if mm else head.pool_cfg
    layers = head.roi_grid_pool_layers_mm if mm else head.roi_grid_pool_layers
    rot_num_id = '' if i == 0 else str(i)
    rois = batch_dict['rois'].clone()
    B = batch_dict['batch_size']
    G = cfg.GRID_SIZE
    xyz = _ref_grid_points(rois, G).view(B, -1, 3)
    pcr, vs = head.point_cloud_range, head.voxel_size
    gc = torch.cat([(xyz[:, :, a:a + 1] - pcr[a]) // vs[a] for a in range(3)], dim=-1)
    batch_idx = rois.new_zeros(B, gc.shape[1], 1)
    for b in range(B):
        batch_idx[b, :, 0] = b
    new_cnt = rois.new_zeros(B).int().fill_(gc.shape[1])
    out = []
    for k, src in enumerate(cfg.FEATURES_SOURCE):
        if src not in SOURCES:
            continue
        stride = batch_dict['multi_scale_3d_strides'][src]
        if not mm:
            j = i
            while 'multi_scale_3d_features' + rot_num_id not in batch_dict:
                j -= 1
                rot_num_id = str(j)
        if batch_dict.get('with_voxel_feature_transform', False):
            sp = batch_dict['multi_scale_3d_features_post'][src]
        elif mm and 'multi_scale_3d_features_mm' + rot_num_id in batch_dict:
            sp = batch_dict['multi_scale_3d_features_mm' + rot_num_id][src]
        else:
            sp = batch_dict['multi_scale_3d_features' + rot_num_id][src]
        c = sp.indices
        dev = c.device
        centres = (c[:, 1:4][:, [2, 1, 0]].float() + 0.5) * (torch.tensor(vs, device=dev).float() * stride) \
            + torch.tensor(pcr[0:3], device=dev).float()
        cnt = centres.new_zeros(B).int()
        for b in range(B):
            cnt[b] = (c[:, 0] == b).sum()
        idx = c.long()
        v2p = -1 * torch.ones(B, *sp.spatial_shape, dtype=torch.int32, device=dev)
        v2p[tuple(idx[:, d] for d in range(idx.shape[1]))] =torch.arange(idx.shape[0], device=dev, dtype=torch.int32)
        nc = torch.cat([batch_idx, gc // stride], dim=-1).int()
        pooled = layers[k](xyz=centres.contiguous(), xyz_batch_cnt=cnt, new_xyz=xyz.contiguous().view(-1, 3),
                           new_xyz_batch_cnt=new_cnt, new_coords=nc.contiguous().view(-1, 4),
                           features=sp.features.contiguous(), voxel2point_indices=v2p)
        out.append(pooled.view(-1, G ** 3, pooled.shape[-1]))
    return torch.cat(out, dim=-1)
