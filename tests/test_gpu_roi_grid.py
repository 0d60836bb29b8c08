"""GPU tests of the RoI grid pooling front end (rules G1-G4 of csrc/roi_grid.cu and virconv_b200/roi_grid.py): the kernel
and the drop-in methods against the reference's own results (tests/golden/roi_grid_ref.npz) and, at full size, against
oracle/roi_grid.py; static-form tensors, a refilled static storage, one map per published tensor, no host sync, CUDA-graph
capture, and the fallback for RoIs that require a gradient."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import roi_grid as o
from oracle import roi_grid_golden as g

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ('A', 'B', 'C')
BRANCHES = (('lidar', 6), ('mm', 4))
SOURCES = ('x_conv3', 'x_conv4')
STRIDES = {'x_conv3': 4, 'x_conv4': 8}


def golden():
    return np.load(os.path.join(os.path.dirname(__file__), 'golden', 'roi_grid_ref.npz'))


def xyz_tol(gold):
    """2 ulp of the largest magnitude, per axis"""
    return 2 * np.spacing(np.abs(gold).max(0).astype(np.float32))


def check_points(xyz, coords, gold_xyz, gold_coords, B, strides, label):
    """xyz within 2 ulp of magnitude; coordinates equal for every point whose golden xyz lies farther than that from a
    cell boundary, and for every point whose xyz is bit-equal to the golden's.  -> the number of the remaining points"""
    tol = xyz_tol(gold_xyz)
    assert (np.abs(xyz - gold_xyz) <= tol).all(), label
    exact = (xyz == gold_xyz).all(1)
    rest = 0
    for k, s in enumerate(strides):
        lo = o.coords(gold_xyz - tol, B, g.PCR, g.VOXEL, s)
        hi = o.coords(gold_xyz + tol, B, g.PCR, g.VOXEL, s)
        safe = (lo == hi).all(1) | exact
        assert np.array_equal(coords[k][safe], gold_coords[k][safe]), (label, s)
        rest += int((~safe).sum())
    print(f'{label}: {rest} of {len(strides) * len(gold_xyz)} coordinates within 2 ulp of a cell boundary')
    return rest


@pytest.mark.parametrize('case', CASES)
@pytest.mark.parametrize('branch,G', BRANCHES)
def test_kernel_matches_golden(lib_built, case, branch, G):
    from virconv_b200.roi_grid import roi_grid_points
    z = golden()
    rois = z[f'{case}.rois']
    strides = [int(s) for s in z['strides']]
    xyz, coords = roi_grid_points(torch.from_numpy(rois).cuda(), G, g.PCR, g.VOXEL, strides)
    pre = f'{case}.{branch}.'
    gold = z[pre + 'global'].reshape(-1, 3)
    check_points(xyz.cpu().numpy(), coords.cpu().numpy(), gold,
                 [g.new_coords(z, pre, k) for k in range(len(strides))], rois.shape[0], strides, pre)


def bench_tensors(seed, B=2, counts=(24000, 9000), C=16, device='cuda'):
    """random x_conv3 / x_conv4 tensors over KITTI's spatial shapes with a VirConv8x-like number of voxels per scene"""
    rng = np.random.default_rng(seed)
    out = {}
    for src, n in zip(SOURCES, counts):
        shape = g.SHAPES[src]
        rows = []
        for b in range(B):
            flat = rng.choice(int(np.prod(shape)), n + 97 * b, replace=False)
            rows.append(np.concatenate([np.full((flat.size, 1), b), np.stack(np.unravel_index(flat, shape), 1)], 1))
        idx = np.concatenate(rows).astype(np.int32)
        idx = idx[rng.permutation(len(idx))]
        feats = rng.standard_normal((len(idx), C)).astype(np.float32)
        out[src] = g.Tensor(torch.from_numpy(feats).to(device), torch.from_numpy(idx).to(device), list(shape), B)
    return out


def kitti_rois(B, N, seed):
    sys.path.insert(0, os.path.join(ROOT, 'profiles'))
    import microbench_part_pool as mb
    return mb.kitti_rois(B, N, seed, torch.device('cuda'))


def test_full_size_matches_oracle(lib_built):
    from virconv_b200 import ops
    from virconv_b200.roi_grid import roi_grid_points, voxel_centers
    rois = kitti_rois(2, 160, 5)
    xyz, coords = roi_grid_points(rois, 6, g.PCR, g.VOXEL, [4, 8])
    assert xyz.shape == (69120, 3) and coords.shape == (2, 69120, 4)
    gold = o.grid_points(rois.cpu().numpy(), 6)
    check_points(xyz.cpu().numpy(), coords.cpu().numpy(), gold, [o.coords(gold, 2, g.PCR, g.VOXEL, s) for s in (4, 8)],
                 2, [4, 8], 'full size')
    for src, t in bench_tensors(1).items():
        idx = t.indices.cpu().numpy()
        assert np.array_equal(voxel_centers(t.indices, STRIDES[src], g.VOXEL, g.PCR).cpu().numpy(),
                              o.voxel_centers(idx, STRIDES[src], g.VOXEL, g.PCR))
        assert np.array_equal(ops.voxel2pinds(t.indices, 2, t.spatial_shape).cpu().numpy(),
                              o.voxel2pinds(idx, 2, t.spatial_shape))


def _fused_layer(C_in, seed=0):
    from virconv_b200.voxel_pool import NeighborVoxelSAModuleMSG
    torch.manual_seed(seed)
    return NeighborVoxelSAModuleMSG(query_ranges=[[2, 2, 2], [4, 4, 4]], radii=[0.4, 0.8], nsamples=[16, 16],
                                    mlps=[[C_in, 32, 32], [C_in, 32, 32]]).cuda()


def _recorder():
    from virconv_b200.voxel_pool import NeighborVoxelSAModuleMSG

    class Recorder(NeighborVoxelSAModuleMSG):
        def __init__(self):
            super().__init__(query_ranges=[[2, 2, 2]], radii=[0.4], nsamples=[16], mlps=[[4, 16, 16]])
            self.calls = []

        def forward(self, **kw):
            self.calls.append(kw)
            return torch.zeros(kw['new_xyz'].shape[0], g.C_FEAT, device=kw['new_xyz'].device)
    return Recorder()


class Head:
    def __init__(self, lidar_layers, mm_layers, grids=(6, 4)):
        ns = __import__('types').SimpleNamespace
        self.pool_cfg = ns(GRID_SIZE=grids[0], FEATURES_SOURCE=list(SOURCES))
        self.pool_cfg_mm = ns(GRID_SIZE=grids[1], FEATURES_SOURCE=list(SOURCES))
        self.roi_grid_pool_layers = lidar_layers
        self.roi_grid_pool_layers_mm = mm_layers
        self.point_cloud_range = g.PCR
        self.voxel_size = list(g.VOXEL)


def _batch(rois, lidar, mm=None):
    bd = {'batch_size': rois.shape[0], 'rois': rois, 'multi_scale_3d_features': lidar,
          'multi_scale_3d_strides': dict(STRIDES)}
    if mm is not None:
        bd['multi_scale_3d_features_mm'] = mm
    return bd


def _golden_tensors(z, case, branch):
    B = z[f'{case}.rois'].shape[0]
    pre = g.tensor_prefix(z, case, branch)
    return {s: g.Tensor(torch.from_numpy(g.features_of(z[f'{pre}s{k}.indices'])).cuda(),
                        torch.from_numpy(z[f'{pre}s{k}.indices']).cuda(), list(g.SHAPES[s]), B)
            for k, s in enumerate(SOURCES)}


@pytest.mark.parametrize('case', CASES)
def test_drop_in_matches_golden(lib_built, case, monkeypatch):
    from virconv_b200 import ops, roi_grid
    z = golden()
    rois = z[f'{case}.rois']
    B = rois.shape[0]
    lidar = _golden_tensors(z, case, 'lidar')
    mm = _golden_tensors(z, case, 'mm') if case == 'A' else None            # B, C: the MM branch reads the LiDAR ones
    head = Head([_recorder(), _recorder()], [_recorder(), _recorder()])
    builds = []
    real = ops.voxel2pinds
    monkeypatch.setattr(ops, 'voxel2pinds', lambda *a, **k: builds.append(1) or real(*a, **k))
    bd = _batch(torch.from_numpy(rois).cuda(), lidar, mm)
    for branch, G, fn, layers in (('lidar', 6, roi_grid.roi_grid_pool, head.roi_grid_pool_layers),
                                  ('mm', 4, roi_grid.roi_grid_pool_mm, head.roi_grid_pool_layers_mm)):
        out = fn(head, bd, 0)
        pre = f'{case}.{branch}.'
        assert tuple(out.shape) == tuple(z[pre + 'out_shape'])
        gold = z[pre + 'global'].reshape(-1, 3)
        coords = [layers[k].calls[0]['new_coords'].cpu().numpy() for k in range(2)]
        check_points(layers[0].calls[0]['new_xyz'].cpu().numpy(), coords, gold,
                     [g.new_coords(z, pre, k) for k in range(2)], B, [4, 8], 'drop-in ' + pre)
        tpre = g.tensor_prefix(z, case, branch)
        feats = lidar if tpre.endswith('lidar.') else mm
        for k in range(2):
            call = layers[k].calls[0]
            assert call['new_xyz'] is layers[0].calls[0]['new_xyz']
            assert call['xyz_batch_cnt'] is None and call['new_xyz_batch_cnt'] is None      # the fused layer reads neither
            assert np.array_equal(call['xyz'].cpu().numpy(), z[f'{tpre}s{k}.xyz'])
            assert np.array_equal(call['voxel2point_indices'].cpu().numpy(), z[f'{tpre}s{k}.v2p'])
            assert torch.equal(call['features'], feats[SOURCES[k]].features)
    assert len(builds) == (4 if case == 'A' else 2)


def static_copy(t, cap):
    """t in static form: capacity-sized, -1 index tail, zero feature tail, device row count .num_rows"""
    n = t.indices.shape[0]
    idx = torch.full((cap, 4), -1, dtype=torch.int32, device=t.indices.device)
    feats = torch.zeros((cap, t.features.shape[1]), dtype=torch.float32, device=t.features.device)
    idx[:n], feats[:n] = t.indices, t.features
    s = g.Tensor(feats, idx, t.spatial_shape, t.batch_size)
    s.num_rows = torch.full((1,), n, dtype=torch.int32, device=idx.device)
    return s


def refill(s, t):
    """write t into the static storage of s (same tensors, new contents)"""
    n = t.indices.shape[0]
    s.indices.fill_(-1)
    s.features.zero_()
    s.indices[:n], s.features[:n] = t.indices, t.features
    s.num_rows.fill_(n)


def _eval_head(C=16):
    head = Head([_fused_layer(C, 1), _fused_layer(C, 2)], [_fused_layer(C, 3), _fused_layer(C, 4)])
    for m in head.roi_grid_pool_layers + head.roi_grid_pool_layers_mm:
        m.eval()
    return head


@pytest.fixture()
def fp32_convs():
    """the pool layer's 1x1 convolutions in fp32: over capacity rows instead of exact rows cuDNN may pick another
    algorithm, and with TF32 the two would differ at TF32's precision"""
    saved = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = saved


def _close(a, b):
    torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5)


def test_static_form_equals_exact(lib_built, fp32_convs):
    from virconv_b200 import roi_grid
    head = _eval_head()
    rois = kitti_rois(2, 160, 7)
    lidar = bench_tensors(2)
    stat = {s: static_copy(t, t.indices.shape[0] + 3001) for s, t in lidar.items()}
    with torch.no_grad():
        for fn in (roi_grid.roi_grid_pool, roi_grid.roi_grid_pool_mm):
            exact = fn(head, _batch(rois, lidar), 0)
            got = fn(head, _batch(rois, stat), 0)
            assert (exact != 0).any()
            _close(got, exact)
    head.roi_grid_pool_layers[0].train()
    with pytest.raises(ValueError, match='static-form'):
        roi_grid.roi_grid_pool(head, _batch(rois, stat), 0)


def test_refilled_static_storage_gives_each_scene_its_result(lib_built, fp32_convs):
    from virconv_b200 import roi_grid
    head = _eval_head()
    rois = kitti_rois(2, 160, 9)
    scenes = [bench_tensors(3), bench_tensors(4, counts=(20000, 8000))]
    cap = 60000
    stat = {s: static_copy(t, cap) for s, t in scenes[0].items()}
    with torch.no_grad():
        outs = []
        for sc in scenes:
            for s, t in sc.items():
                refill(stat[s], t)
            outs.append(roi_grid.roi_grid_pool(head, _batch(rois, stat), 0))
        for sc, got in zip(scenes, outs):
            _close(got, roi_grid.roi_grid_pool(head, _batch(rois, sc), 0))
    assert not torch.equal(outs[0], outs[1])


def test_map_built_once_per_published_tensor(lib_built, monkeypatch):
    """VirConv-T's training step: three stages, each calling both branches with i = 0 (ted_head.py:794-795), over the
    LiDAR and the MM tensors of x_conv3 / x_conv4: four maps, where the reference builds twelve"""
    from virconv_b200 import ops, roi_grid
    head = _eval_head()
    lidar, mm = bench_tensors(5), bench_tensors(6)
    builds = []
    real = ops.voxel2pinds
    monkeypatch.setattr(ops, 'voxel2pinds', lambda *a, **k: builds.append(1) or real(*a, **k))
    bd = _batch(kitti_rois(2, 160, 11), lidar, mm)
    with torch.no_grad():
        for stage in range(3):
            bd['rois'] = kitti_rois(2, 160, 20 + stage)
            roi_grid.roi_grid_pool(head, bd, 0)
            roi_grid.roi_grid_pool_mm(head, bd, 0)
    assert len(builds) == 4


def test_no_host_sync(lib_built):
    from virconv_b200 import roi_grid
    head = Head([_fused_layer(16, 1), _fused_layer(16, 2)], [_fused_layer(16, 3), _fused_layer(16, 4)])
    rois = kitti_rois(2, 160, 13)
    lidar = bench_tensors(7)
    stat = {s: static_copy(t, t.indices.shape[0] + 100) for s, t in lidar.items()}
    for m in head.roi_grid_pool_layers_mm:
        m.eval()
    roi_grid.roi_grid_pool(head, _batch(rois, lidar), 0)          # warm-up: library load, allocator
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = roi_grid.roi_grid_pool(head, _batch(rois, lidar), 0)                 # training mode, exact tensors
        out.sum().backward()
        roi_grid.roi_grid_pool_mm(head, _batch(rois, stat), 0)                    # eval mode, static form
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_cuda_graph_replays_equal_eager(lib_built):
    from virconv_b200 import roi_grid
    head = _eval_head()
    rois = kitti_rois(2, 160, 15)
    lidar = bench_tensors(8)
    mm = {s: static_copy(t, t.indices.shape[0] + 500) for s, t in bench_tensors(9).items()}

    def step():
        bd = _batch(rois, lidar, mm)
        with torch.no_grad():
            return roi_grid.roi_grid_pool(head, bd, 0), roi_grid.roi_grid_pool_mm(head, bd, 0)

    eager = [t.clone() for t in step()]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    for _ in range(3):
        for t in outs:
            t.fill_(float('nan'))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(outs[0], eager[0]) and torch.equal(outs[1], eager[1])


def test_rois_with_gradient_take_the_fallback(lib_built, monkeypatch):
    from virconv_b200 import roi_grid
    head = _eval_head()
    calls = []
    monkeypatch.setattr(roi_grid, '_reference_roi_grid_pool', lambda s, b, i: calls.append(b['rois']) or 'ref')
    monkeypatch.setattr(roi_grid, '_reference_roi_grid_pool_mm', lambda s, b, i: calls.append(b['rois']) or 'ref_mm')
    rois = kitti_rois(2, 20, 17).requires_grad_()
    bd = _batch(rois, bench_tensors(10))
    assert roi_grid.roi_grid_pool(head, bd, 0) == 'ref' and roi_grid.roi_grid_pool_mm(head, bd, 0) == 'ref_mm'
    assert calls[0] is rois and calls[1] is rois
