"""Record what the reference's OWN `TEDMHead.roi_grid_pool` and `roi_grid_pool_mm` (ted_head.py:450-673, with
`common_utils.get_voxel_centers` and `spconv_utils.generate_voxel2pinds`) compute, as tests/golden/roi_grid_ref.npz.
Needs the reference's sources (imported through virconv_b200.reference_env); the fixture it writes is committed, so the
tests need neither.  The methods run on the CPU on a stand-in head (the reference class without its network) whose pool
layers record the seven arguments they are called with and return zeros.

KITTI's POINT_CLOUD_RANGE (an np.float32 array, as dataset.py:35 builds it) and VOXEL_SIZE (Python floats), the
x_conv3 / x_conv4 sources at strides 4 / 8 on their KITTI spatial shapes, with a few thousand random voxels per scene.
Per case, keys `{case}.*`:
  rois [B, N, 7]; `lidar.` / `mm.` (G = 6 / 4): global and local grid points of get_global_grid_points_of_roi, and of
  the whole method call new_xyz_batch_cnt, the output shape and, per source k, new_coords (compacted: read them with
  local() and new_coords()).  Per published
  tensor (`lidar.`, and `mm.` where the MM branch has its own: tensor_prefix()) and source k: the indices
  `s{k}.indices` and what the pool layer received for it, `s{k}.xyz`, `s{k}.xyz_batch_cnt` and the map `s{k}.v2p`.
  Not stored, but asserted by make(): the new_xyz the pool layers receive (the global grid points viewed as [-1, 3]),
  the features (the tensor's own, features_of(indices)), and the MM call's records where it reads the LiDAR tensors
  (equal to the LiDAR call's).
Cases:
  A — B = 1, N = 160: random RoIs over and beyond the range (below it: negative voxel coordinates), headings 0, +-pi/2,
      pi; zero-size RoIs whose every grid point is its centre, placed exactly on cell boundaries (multiples of the
      voxel size that are exact in float32, which are boundaries at strides 4 and 8 too), below and above the range;
      heading-0 RoIs with dyadic centres and sizes (exact grid points); the MM branch reads its own tensors;
  B — B = 2, N = 50: random RoIs, zero rows at the end of scene 1; the MM branch falls back to the LiDAR tensors;
  C — B = 1, N = 1.

    python -m oracle.roi_grid_golden REFERENCE_ROOT [OUT_DIR]
"""
from __future__ import annotations

import os
import sys

import numpy as np

SEED = 53
PCR = np.array([0, -40, -3, 70.4, 40, 1], dtype=np.float32)
VOXEL = [0.05, 0.05, 0.1]
STRIDES = {'x_conv3': 4, 'x_conv4': 8}
SHAPES = {'x_conv3': (11, 400, 352), 'x_conv4': (5, 200, 176)}
SOURCES = ('x_conv3', 'x_conv4')
C_FEAT = 4
GRIDS = {'lidar': 6, 'mm': 4}
CASES = ('A', 'B', 'C')
f32 = np.float32


def random_rois(rng, shape):
    r = np.zeros((*shape, 7), np.float32)
    r[..., 0] = rng.uniform(-3.0, 74.0, shape)
    r[..., 1] = rng.uniform(-43.0, 43.0, shape)
    r[..., 2] = rng.uniform(-3.5, 1.5, shape)
    r[..., 3] = rng.uniform(0.5, 4.6, shape)
    r[..., 4] = rng.uniform(0.5, 1.9, shape)
    r[..., 5] = rng.uniform(0.8, 1.7, shape)
    r[..., 6] = rng.uniform(-np.pi, np.pi, shape)
    return r


def boundary_values(axis):
    """world coordinates on cell boundaries: range + voxel * 2^p, exact in float32 (so is the subtraction of the range)"""
    v, lo = f32(VOXEL[axis]), f32(PCR[axis])
    out = []
    for p in range(0, 11):
        x = f32(v * f32(2 ** p))
        w = f32(x + lo)
        if f32(w - lo) == x and w <= PCR[axis + 3]:
            out.append(w)
    return np.array(out, np.float32)


def case_a(rng):
    r = random_rois(rng, (1, 160))[0]
    r[0:4, 6] = [0.0, np.pi / 2, -np.pi / 2, np.pi]
    bx, by, bz = boundary_values(0), boundary_values(1), boundary_values(2)
    for n in range(4, 40):                                            # zero-size RoIs on cell boundaries
        r[n, 0], r[n, 1], r[n, 2] = bx[n % len(bx)], by[(3 * n) % len(by)], bz[n % len(bz)]
        r[n, 3:6] = 0
        r[n, 6] = [0.0, np.pi / 2, -np.pi / 2, np.pi][n % 4]
    r[40:44, 0] = [-0.8, -3.2, 75.0, 0.0]                             # zero-size, below / beyond the range
    r[40:44, 1] = [-41.6, 44.8, -40.0, 41.6]
    r[40:44, 2] = [-3.2, -4.6, 1.0, -3.0]
    r[40:44, 3:6] = 0
    for n in range(44, 60):                                           # heading 0, dyadic centres and sizes
        r[n, 0] = rng.integers(-16, 600) / 8
        r[n, 1] = rng.integers(-330, 330) / 8
        r[n, 2] = rng.integers(-28, 8) / 8
        r[n, 3:6] = rng.integers(1, 9, 3) * 0.75     # G * 2^-k for G = 6 and 4: (i + 0.5) / G * size is dyadic
        r[n, 6] = 0.0
    r[60:64, 0] = [-2.5, 72.5, 35.0, 35.0]                            # whole RoIs below / beyond the range
    r[60:64, 1] = [0.0, 0.0, -42.0, 42.0]
    return r[None]


def case_b(rng):
    r = random_rois(rng, (2, 50))
    r[0, :3, 6] = [0.0, np.pi, -np.pi / 2]
    r[1, 45:] = 0
    return r


def case_c(rng):
    return random_rois(rng, (1, 1))


class Tensor:
    """the attributes of a spconv SparseConvTensor the methods read"""

    def __init__(self, features, indices, spatial_shape, batch_size):
        self.features, self.indices, self.spatial_shape, self.batch_size = features, indices, spatial_shape, batch_size


def sparse(rng, B, src):
    import torch
    shape = SHAPES[src]
    rows = []
    for b in range(B):
        n = int(rng.integers(400, 800))
        flat = rng.choice(int(np.prod(shape)), n, replace=False)
        zyx = np.stack(np.unravel_index(flat, shape), 1)
        rows.append(np.concatenate([np.full((n, 1), b), zyx], 1))
    idx = np.concatenate(rows).astype(np.int32)
    idx = idx[rng.permutation(idx.shape[0])]                          # rows of the scenes interleaved
    return Tensor(torch.from_numpy(features_of(idx)), torch.from_numpy(idx), list(shape), B)


def features_of(idx):
    """[n, C_FEAT] dyadic float32 features, a function of the voxel indices [n, 4] (so the fixture need not store them)"""
    idx = np.asarray(idx, np.int64)
    v = idx[:, 1:2] * 7 + idx[:, 2:3] * 3 + idx[:, 3:4] * 5 + idx[:, 0:1] + np.arange(C_FEAT) * 11
    return ((v % 129 - 64) / 16).astype(np.float32)


def local(z, pre):
    """the local grid points [B * N, G^3, 3] of get_global_grid_points_of_roi from `{pre}local_axis` [B * N, G, 3]"""
    la = z[pre + 'local_axis']
    G = la.shape[1]
    i, j, k = (a.reshape(-1) for a in np.meshgrid(np.arange(G), np.arange(G), np.arange(G), indexing='ij'))
    return np.stack([la[:, i, 0], la[:, j, 1], la[:, k, 2]], -1)


def new_coords(z, pre, k):
    """the new_coords [M, 4] int32 (b, x, y, z) the pool layer of source k received, from `{pre}s{k}.xyz_coords`
    [M, 3] int16 (rows scene-major, M / B per scene)"""
    xyz = z[f'{pre}s{k}.xyz_coords'].astype(np.int32)
    B = z[pre.split('.')[0] + '.rois'].shape[0]
    b = np.repeat(np.arange(B, dtype=np.int32), xyz.shape[0] // B)
    return np.concatenate([b[:, None], xyz], 1)


def tensor_prefix(z, case, branch):
    """the key prefix of the published tensor the `branch` call of `case` reads"""
    return f'{case}.mm.' if branch == 'mm' and f'{case}.mm.s0.indices' in z else f'{case}.lidar.'


def head_and_layers():
    import torch
    from pcdet.models.roi_heads import ted_head
    from virconv_b200.reference_env import EasyDict

    class Recorder(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.calls = []

        def forward(self, **kw):
            self.calls.append({k: (v.clone() if torch.is_tensor(v) else v) for k, v in kw.items()})
            return torch.zeros(kw['new_xyz'].shape[0], C_FEAT)

    head = ted_head.TEDMHead.__new__(ted_head.TEDMHead)
    torch.nn.Module.__init__(head)
    head.pool_cfg = EasyDict(GRID_SIZE=GRIDS['lidar'], FEATURES_SOURCE=list(SOURCES))
    head.pool_cfg_mm = EasyDict(GRID_SIZE=GRIDS['mm'], FEATURES_SOURCE=list(SOURCES))
    head.roi_grid_pool_layers = torch.nn.ModuleList([Recorder() for _ in SOURCES])
    head.roi_grid_pool_layers_mm = torch.nn.ModuleList([Recorder() for _ in SOURCES])
    head.point_cloud_range = PCR
    head.voxel_size = list(VOXEL)
    return head


def run_case(rng, name, rois, mm_own):
    import torch
    B = rois.shape[0]
    head = head_and_layers()
    lidar = {s: sparse(rng, B, s) for s in SOURCES}
    bd = {'batch_size': B, 'rois': torch.from_numpy(rois), 'multi_scale_3d_features': lidar,
          'multi_scale_3d_strides': dict(STRIDES)}
    mm = None
    if mm_own:
        mm = {s: sparse(rng, B, s) for s in SOURCES}
        bd['multi_scale_3d_features_mm'] = mm
    res = {f'{name}.rois': rois}
    for branch, method, layers, feats in (
            ('lidar', head.roi_grid_pool, head.roi_grid_pool_layers, lidar),
            ('mm', head.roi_grid_pool_mm, head.roi_grid_pool_layers_mm, mm or lidar)):
        G = GRIDS[branch]
        glob, loc = head.get_global_grid_points_of_roi(torch.from_numpy(rois), grid_size=G)
        out = method(bd, 0)
        pre = f'{name}.{branch}.'
        res[pre + 'global'] = glob.numpy()
        # the local points are separable: the value along axis a depends on the RoI and that axis' grid index only
        res[pre + 'local_axis'] = loc.numpy()[:, [(i * G + i) * G + i for i in range(G)], :]
        assert np.array_equal(local(res, pre), loc.numpy())
        res[pre + 'out_shape'] = np.array(out.shape)
        for k, s in enumerate(SOURCES):
            (call,) = layers[k].calls
            if k == 0:
                res[pre + 'new_xyz_batch_cnt'] = call['new_xyz_batch_cnt'].numpy()
            assert np.array_equal(res[pre + 'global'].reshape(-1, 3), call['new_xyz'].numpy())     # new_xyz: not stored
            nc = call['new_coords'].numpy()
            assert np.abs(nc[:, 1:]).max() < 2 ** 15
            res[f'{pre}s{k}.xyz_coords'] = nc[:, 1:].astype(np.int16)      # the batch column is the scene of the row
            assert np.array_equal(new_coords(res, pre, k), nc)
            assert torch.equal(call['features'], feats[s].features)
            rec = {'xyz': call['xyz'].numpy(), 'xyz_batch_cnt': call['xyz_batch_cnt'].numpy(),
                   'indices': feats[s].indices.numpy(), 'v2p': call['voxel2point_indices'].numpy()}
            if branch == 'mm' and mm is None:          # the LiDAR tensor again: the same records
                for key, v in rec.items():
                    assert np.array_equal(v, res[f'{name}.lidar.s{k}.{key}']), key
            else:
                res.update({f'{pre}s{k}.{key}': v for key, v in rec.items()})
    return res


def make(reference_root, out_dir):
    import virconv_b200.reference_env as renv
    renv.install(reference_root=reference_root)
    rng = np.random.default_rng(SEED)
    res = {'pcr': PCR, 'voxel': np.array(VOXEL), 'strides': np.array([STRIDES[s] for s in SOURCES]),
           'grids': np.array([GRIDS['lidar'], GRIDS['mm']])}
    for name, fn, mm_own in (('A', case_a, True), ('B', case_b, False), ('C', case_c, False)):
        res.update(run_case(rng, name, fn(rng), mm_own))
        print(name, res[f'{name}.rois'].shape)
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'roi_grid_ref.npz')
    np.savez_compressed(path, **res)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    make(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else os.path.join(root, 'tests', 'golden'))
