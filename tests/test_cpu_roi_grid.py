"""The RoI grid pooling front end without a GPU: the float32 restatement oracle/roi_grid.py against the reference's own
`TEDMHead.roi_grid_pool` / `roi_grid_pool_mm` (tests/golden/roi_grid_ref.npz, recorded by oracle/roi_grid_golden.py),
the fix-up cases of torch's float floor division, the coverage of the golden cases, the library's new symbol, the
drop-ins' fallbacks and feature-dict choice, and — where the reference's sources exist — the VirConv-T detector built
with `reference_env.install(use_fused_roi_grid=True)`."""
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import roi_grid as o
from oracle import roi_grid_golden as g
from test_cpu_part_pool import _build_detector
from test_cpu_voxel_pool import _restore_modules, need_ref

CASES = ('A', 'B', 'C')
BRANCHES = (('lidar', 6), ('mm', 4))


def golden():
    return np.load(os.path.join(os.path.dirname(__file__), 'golden', 'roi_grid_ref.npz'))


def xyz_tol(gold):
    """2 ulp of the largest magnitude, per axis"""
    return 2 * np.spacing(np.abs(gold).max(0).astype(np.float32))


@pytest.mark.parametrize('case', CASES)
@pytest.mark.parametrize('branch,G', BRANCHES)
def test_oracle_matches_reference(case, branch, G):
    z = golden()
    pcr, vs = z['pcr'], [float(v) for v in z['voxel']]
    rois = z[f'{case}.rois']
    pre = f'{case}.{branch}.'
    gold = z[pre + 'global'].reshape(-1, 3)
    assert np.array_equal(o.local_points(rois.reshape(-1, 7), G), g.local(z, pre))
    assert (np.abs(o.grid_points(rois, G) - gold) <= xyz_tol(gold)).all()
    assert tuple(z[pre + 'out_shape']) == (rois.shape[0] * rois.shape[1], G ** 3, 2 * g.C_FEAT)
    assert (z[pre + 'new_xyz_batch_cnt'] == rois.shape[1] * G ** 3).all()
    for k, stride in enumerate(z['strides']):
        assert np.array_equal(o.coords(gold, rois.shape[0], pcr, vs, int(stride)), g.new_coords(z, pre, k))
        s = f'{g.tensor_prefix(z, case, branch)}s{k}.'
        idx = z[s + 'indices']
        assert np.array_equal(o.voxel_centers(idx, int(stride), vs, pcr), z[s + 'xyz'])
        v2p = z[s + 'v2p']
        assert np.array_equal(o.voxel2pinds(idx, rois.shape[0], v2p.shape[1:]), v2p)
        assert np.array_equal(z[s + 'xyz_batch_cnt'], np.bincount(idx[:, 0], minlength=rois.shape[0]))


def test_div_floor_fixups():
    """inputs where floor(a / b) is off by one and torch's div_floor_floating is not (found with torch on the CPU)"""
    a = np.array([0.45, -0.95000005, 0.9, -1.9000001, -0.0, 0.0, -1e-8, 1.6, -1.6], np.float32)
    b = np.array([0.05, 0.05, 0.1, 0.1, 0.05, 0.05, 0.05, 0.1, 0.1], np.float32)
    want = np.array([8, -20, 8, -20, -0.0, 0.0, -1, 16, -16], np.float32)
    assert np.array_equal(np.floor(a / b)[:4], [9, -19, 9, -19])                 # the naive rule differs
    got = o.div_floor(a, b)
    assert np.array_equal(got, want) and np.array_equal(np.signbit(got), np.signbit(want))
    assert np.array_equal(got, (torch.from_numpy(a) // torch.from_numpy(b)).numpy())


def test_golden_covers_edge_cases():
    z = golden()
    shapes = {z[f'{c}.rois'].shape[:2] for c in CASES}
    assert {s[0] for s in shapes} == {1, 2} and {s[1] for s in shapes} == {1, 50, 160}
    rois = z['A.rois'][0]
    for h in (0.0, np.pi / 2, -np.pi / 2, np.pi):
        assert (rois[:, 6] == np.float32(h)).any(), h
    assert ((rois[:, 3:6] == 0).all(1)).sum() >= 30                               # zero-size RoIs
    pcr, vs = z['pcr'], [float(v) for v in z['voxel']]
    gold = z['A.lidar.global'].reshape(-1, 3)
    rel = gold - pcr[:3]
    v = o.div_floor(rel, np.asarray(vs, np.float32))
    on_cell = (v * np.asarray(vs, np.float32) == rel)                             # exactly on a cell boundary
    assert on_cell.all(1).sum() > 100
    for stride in z['strides']:
        assert (on_cell.all(1) & (np.fmod(v, stride) == 0).all(1)).sum() > 50      # ... and a stride boundary
    c = g.new_coords(z, 'A.lidar.', 0)
    assert (c[:, 1:] < 0).any() and (gold < pcr[:3]).any() and (gold > pcr[3:]).any()
    assert (z['B.rois'][1, 45:] == 0).all()


def test_new_symbol_declared(lib_built):
    from virconv_b200 import _lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include',
                               'virconv_b200.h')).read()
    assert 'vc_roi_grid_points' in _lib.SIGNATURES and ' vc_roi_grid_points(' in header
    lib = _lib.load()
    p = ctypes.c_void_p(16)     # never dereferenced: every call below returns before a launch
    f3 = _lib.host_f32([0.0, -40.0, -3.0])
    call = lambda B, N, ld, G, st: lib.vc_roi_grid_points(p, B, N, ld, G, f3, f3, _lib.host_i32(st), len(st), p, p,  # noqa
                                                          None)
    assert call(2, 160, 7, 6, [4, 8, 1, 2, 16]) == -4           # VC_ERR_UNSUPPORTED: more than 4 sources
    assert call(2, 160, 6, 6, [4]) == -1 and call(2, 160, 7, 0, [4]) == -1 and call(2, 160, 7, 6, [0]) == -1
    assert call(0, 160, 7, 6, [4, 8]) == 0 and call(2, 0, 7, 6, [4, 8]) == 0


def _head():
    cfg = types.SimpleNamespace(GRID_SIZE=6, FEATURES_SOURCE=['x_conv3', 'x_conv4'])
    return types.SimpleNamespace(pool_cfg=cfg, pool_cfg_mm=types.SimpleNamespace(GRID_SIZE=4, FEATURES_SOURCE=['x_conv3']),
                                 roi_grid_pool_layers=[torch.nn.Identity(), torch.nn.Identity()],
                                 roi_grid_pool_layers_mm=[torch.nn.Identity()], point_cloud_range=g.PCR,
                                 voxel_size=list(g.VOXEL))


def test_fallbacks_go_to_reference_method(monkeypatch):
    """a pool layer that is not the fused class, RoIs with a gradient, a source other than x_conv1..4"""
    from virconv_b200 import roi_grid as rg
    from virconv_b200.voxel_pool import NeighborVoxelSAModuleMSG
    head = _head()
    bd = {'rois': torch.zeros(1, 3, 7), 'batch_size': 1}
    monkeypatch.setattr(rg, '_reference_roi_grid_pool', None)
    with pytest.raises(RuntimeError, match='reference method'):
        rg.roi_grid_pool(head, bd, 0)
    calls = []
    monkeypatch.setattr(rg, '_reference_roi_grid_pool', lambda s, b, i: calls.append((s, b, i)) or 'ref')
    monkeypatch.setattr(rg, '_reference_roi_grid_pool_mm', lambda s, b, i: calls.append((s, b, i)) or 'ref_mm')
    assert rg.roi_grid_pool(head, bd, 2) == 'ref' and calls[-1] == (head, bd, 2)
    assert rg.roi_grid_pool_mm(head, bd, 1) == 'ref_mm'
    fused = NeighborVoxelSAModuleMSG(query_ranges=[[2, 2, 2]], radii=[0.4], nsamples=[16], mlps=[[4, 16, 16]])
    head.roi_grid_pool_layers = [fused, fused]
    head.roi_grid_pool_layers_mm = [fused]
    bd['rois'] = torch.zeros(1, 3, 7, requires_grad=True)
    assert rg.roi_grid_pool(head, bd, 0) == 'ref' and rg.roi_grid_pool_mm(head, bd, 0) == 'ref_mm'
    bd['rois'] = torch.zeros(1, 3, 7)
    head.pool_cfg.FEATURES_SOURCE = ['x_conv3', 'bev']
    assert rg.roi_grid_pool(head, bd, 0) == 'ref'
    assert len(calls) == 5


def test_feature_dict_choice():
    from virconv_b200 import roi_grid as rg
    bd = {'multi_scale_3d_features': 'L0', 'multi_scale_3d_features1': 'L1', 'multi_scale_3d_features_mm': 'M0'}
    assert rg._lidar_features(bd, 0) == 'L0' and rg._lidar_features(bd, 1) == 'L1'
    assert rg._lidar_features(bd, 2) == 'L1'
    with pytest.raises(KeyError):             # the reference's loop falls back to '0', not '': it would never end
        rg._lidar_features({'multi_scale_3d_features': 'L0'}, 1)
    bd['multi_scale_3d_features0'] = 'L00'
    assert rg._lidar_features(bd, 3) == 'L1' and rg._lidar_features({'multi_scale_3d_features0': 'x'}, 2) == 'x'
    with pytest.raises(KeyError):
        rg._lidar_features({'multi_scale_3d_features1': 'x'}, 0)
    assert rg._mm_features(bd, 0) == 'M0' and rg._mm_features(bd, 1) == 'L1'       # VirConv-L: the LiDAR tensors
    bd['with_voxel_feature_transform'] = True
    bd['multi_scale_3d_features_post'] = 'P'
    assert rg._lidar_features(bd, 1) == 'P' and rg._mm_features(bd, 1) == 'P'


def test_rejects_cpu_rois():
    from virconv_b200._lib import VirConvLibraryError
    from virconv_b200.roi_grid import roi_grid_points
    with pytest.raises(VirConvLibraryError):
        roi_grid_points(torch.zeros(1, 3, 7), 6, g.PCR, g.VOXEL, [4, 8])


@need_ref
def test_virconv_t_head_uses_fused_roi_grid(monkeypatch):
    from virconv_b200 import roi_grid as rg
    saved = dict(sys.modules)
    try:
        model = _build_detector(monkeypatch, 'VirConv-T.yaml')
        keys_default = list(model.state_dict())
        assert type(model.roi_head).roi_grid_pool is not rg.roi_grid_pool
        assert type(model.roi_head).roi_grid_pool_mm is not rg.roi_grid_pool_mm
    finally:
        _restore_modules(saved)
    monkeypatch.setattr(rg, '_reference_roi_grid_pool', None)
    monkeypatch.setattr(rg, '_reference_roi_grid_pool_mm', None)
    try:
        model = _build_detector(monkeypatch, 'VirConv-T.yaml', use_fused_roi_grid=True, use_fused_roi_pool=True)
        head = model.roi_head
        assert type(head).__name__ == 'TEDMHead'
        assert type(head).roi_grid_pool is rg.roi_grid_pool and type(head).roi_grid_pool_mm is rg.roi_grid_pool_mm
        for ref in (rg._reference_roi_grid_pool, rg._reference_roi_grid_pool_mm):
            assert ref is not None and ref.__module__ == 'pcdet.models.roi_heads.ted_head'
        bd = {'rois': torch.zeros(1, 2, 7)}
        assert rg._fused_ok(bd, head.pool_cfg, head.roi_grid_pool_layers)
        assert rg._fused_ok(bd, head.pool_cfg_mm, head.roi_grid_pool_layers_mm)
        assert list(model.state_dict()) == keys_default
    finally:
        _restore_modules(saved)
