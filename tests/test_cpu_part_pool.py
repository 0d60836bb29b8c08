"""Part-score RoI pooling without a GPU: the float64 restatement oracle/part_pool.py against the reference's own
`TEDMHead.obtain_conf_preds` and its part-map gradient (tests/golden/part_pool_ref.npz, recorded by
oracle/part_pool_golden.py), the coverage of the golden cases, the library's new symbols and limits, the Python
operator's device check and fallback, and — where the reference's sources exist — the VirConv-T detector built with
`reference_env.install(use_fused_part_pool=True)`."""
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import part_pool as o
from oracle import part_pool_golden as g
from test_cpu_voxel_pool import REF, _restore_modules, need_ref

SYMS = ('vc_part_pool_fwd', 'vc_part_pool_bwd_ws_bytes', 'vc_part_pool_bwd')
CASES = ('A', 'B', 'C', 'D')


def golden():
    return np.load(os.path.join(os.path.dirname(__file__), 'golden', 'part_pool_ref.npz'))


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _geo_dict(z, case):
    S, off, scale, stride = g.geom_of(z, case)
    H, W = z[f'{case}.parts'].shape[2:]
    return dict(offsets=off, stride=stride, H=H, W=W)


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_reference(case):
    z = golden()
    S, off, scale, _ = g.geom_of(z, case)
    parts, rois, grad = z[f'{case}.parts'], z[f'{case}.rois'], z[f'{case}.g']
    out = o.forward(parts, rois, S, off, scale)
    d = o.backward(rois, grad, parts.shape, S, off, scale)
    assert out.shape == z[f'{case}.out'].shape == (rois.shape[0] * rois.shape[1], 1)
    assert _rel(out, z[f'{case}.out']) < 1e-10 and _rel(d, z[f'{case}.dparts']) < 1e-10
    # fp32: the coordinates round in fp32 in the model
    assert _rel(out, z[f'f32.{case}.out']) < 1e-4 and _rel(d, z[f'f32.{case}.dparts']) < 1e-4
    assert np.array_equal(d != 0, z[f'{case}.dparts'] != 0)


@pytest.mark.parametrize('case', CASES)
def test_golden_samples_are_unambiguous(case):
    z = golden()
    rois = z[f'{case}.rois']
    assert g.sample_ok(rois.reshape(-1, rois.shape[-1]).astype(np.float64), _geo_dict(z, case)).all()


def test_golden_covers_edge_cases():
    z = golden()
    shapes = {c: z[f'{c}.rois'].shape[:2] for c in CASES}
    assert {s[0] for s in shapes.values()} == {1, 2} and {s[1] for s in shapes.values()} == {1, 50, 160}
    rois = z['A.rois'][0]
    S, off, scale, _ = g.geom_of(z, 'A')
    H, W = z['A.parts'].shape[2:]
    ix, iy = o.positions(rois, S, off, scale, H, W)
    x0, y0 = np.floor(ix), np.floor(iy)
    inside = (x0 >= 0) & (x0 + 1 <= W - 1) & (y0 >= 0) & (y0 + 1 <= H - 1)      # all four taps in the map
    none = (x0 + 1 < 0) | (x0 > W - 1) | (y0 + 1 < 0) | (y0 > H - 1)             # no tap in the map
    nonzero = np.abs(rois).sum(1) > 0
    assert (inside.all(1) & nonzero).any()
    assert (none.all(1) & nonzero).any()                                         # fully outside
    for cross in (x0 < 0, x0 + 1 > W - 1, y0 < 0, y0 + 1 > H - 1):                # straddling each border
        assert (cross.any(1) & inside.any(1)).any()
    heads = rois[:, 6]
    for h in (0.0, np.pi / 2, -np.pi / 2, np.pi):
        assert (heads == np.float32(h)).any(), h
    assert ((heads != 0) & (np.abs(np.abs(heads) - np.float32(np.pi / 2)) > 1e-3) & (np.abs(heads) < 3.1)).sum() > 50
    assert ((rois[:, 3] == 0) & (rois[:, 4] == 0) & nonzero).any()               # zero-size boxes
    assert (~nonzero).sum() >= 20 and (~nonzero[-20:]).all()                     # proposal padding rows
    u, c = np.unique(rois[nonzero], axis=0, return_counts=True)
    assert c.max() >= 20                                                         # one box many times: taps collide
    # dyadic case: samples exactly on integer and half-integer pixel coordinates, in the map and at its borders
    S, off, scale, _ = g.geom_of(z, 'D')
    H, W = z['D.parts'].shape[2:]
    ix, iy = o.positions(z['D.rois'], S, off, scale, H, W)
    for a in (ix, iy):
        assert (a == np.round(a)).sum() > 100 and (a - np.floor(a) == 0.5).sum() > 100
    assert ((ix == -0.5) | (ix == W - 0.5) | (ix == W - 1)).any()
    assert (z['D.dparts'] != 0).any()


def test_new_symbols_declared():
    from virconv_b200 import _lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include',
                               'virconv_b200.h')).read()
    for sym in SYMS:
        assert sym in _lib.SIGNATURES
        assert f' {sym}(' in header


def test_library_exports_new_symbols(lib_built):
    lib = ctypes.CDLL(lib_built)
    for sym in SYMS:
        assert hasattr(lib, sym)


def test_library_limits(lib_built):
    """arguments the C entry points refuse before they enqueue anything"""
    from virconv_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(16)   # never dereferenced: every call below returns before a launch
    fwd = lambda B, N, ld, S: lib.vc_part_pool_fwd(p, p, B, N, ld, S, 40, 36, 0.0, 40.0, 2.5, p, None)   # noqa: E731
    bwd = lambda B, N, ld, S: lib.vc_part_pool_bwd(p, p, B, N, ld, S, 40, 36, 0.0, 40.0, 2.5, p, None, 0,  # noqa: E731
                                                   None)
    for f in (fwd, bwd):
        assert f(2, 1025, 7, 7) == -4                 # VC_ERR_UNSUPPORTED: more RoIs than VC_PART_POOL_MAX_ROIS
        assert f(2, 160, 7, 17) == -4 and f(2, 160, 7, 1) == -4
        assert f(2, 160, 6, 7) == -1                  # VC_ERR_INVALID: a RoI row shorter than 7
        assert f(-1, 160, 7, 7) == -1
        assert f(0, 160, 7, 7) == 0                   # no scene: nothing to do
    assert fwd(2, 0, 7, 7) == 0
    assert lib.vc_part_pool_bwd_ws_bytes(2, 160, 7) == 0


def test_operator_rejects_cpu_tensors():
    from virconv_b200._lib import VirConvLibraryError
    from virconv_b200.part_pool import obtain_conf_preds, part_pool
    parts, rois = torch.zeros(1, 49, 8, 8), torch.zeros(1, 3, 7)
    with pytest.raises(VirConvLibraryError):
        part_pool(parts, rois, 7, (0.0, 40.0), 2.5)
    head = types.SimpleNamespace(grid_offsets=[0.0, 40.0], featmap_stride=0.4)
    with pytest.raises(VirConvLibraryError):
        obtain_conf_preds(head, parts, rois)


def test_rois_with_gradient_go_to_reference_method(monkeypatch):
    from virconv_b200 import part_pool
    head = types.SimpleNamespace(grid_offsets=[0.0, 40.0], featmap_stride=0.4)
    parts, rois = torch.zeros(1, 49, 8, 8), torch.zeros(1, 3, 7, requires_grad=True)
    monkeypatch.setattr(part_pool, '_reference_obtain_conf_preds', None)
    with pytest.raises(RuntimeError, match='reference method'):
        part_pool.obtain_conf_preds(head, parts, rois)
    calls = []
    monkeypatch.setattr(part_pool, '_reference_obtain_conf_preds', lambda s, a, b: calls.append((s, a, b)) or 'ref')
    assert part_pool.obtain_conf_preds(head, parts, rois) == 'ref'
    assert calls[0][0] is head and calls[0][2] is rois


def _build_detector(monkeypatch, yaml_name, **install_kw):
    import virconv_b200.reference_env as renv
    renv.install(reference_root=REF, use_fused_backbones=True, **install_kw)
    from pcdet.config import cfg, cfg_from_yaml_file
    from pcdet.models import build_network
    cwd = os.getcwd()
    os.chdir(os.path.join(REF, 'tools'))
    try:
        cfg_from_yaml_file(os.path.join('cfgs', 'models', 'kitti', yaml_name), cfg)
    finally:
        os.chdir(cwd)
    pcr = np.array(cfg.DATA_CONFIG.POINT_CLOUD_RANGE, dtype=np.float32)
    vs = [p.VOXEL_SIZE for p in cfg.DATA_CONFIG.DATA_PROCESSOR if p.NAME == 'transform_points_to_voxels'][0]
    grid = np.round((pcr[3:6] - pcr[0:3]) / np.array(vs)).astype(np.int64)
    ds = types.SimpleNamespace(class_names=cfg.CLASS_NAMES, point_feature_encoder=types.SimpleNamespace(num_point_features=8),
                               grid_size=grid, voxel_size=vs, point_cloud_range=pcr, depth_downsample_factor=None,
                               test_flip=False, rot_num=1)
    monkeypatch.setattr(torch.Tensor, 'cuda', lambda self, *a, **k: self)     # the anchor generator calls .cuda()
    return build_network(model_cfg=cfg.MODEL, num_class=len(cfg.CLASS_NAMES), dataset=ds)


@need_ref
def test_virconv_t_head_uses_fused_part_pool(monkeypatch):
    from virconv_b200 import part_pool
    saved = dict(sys.modules)
    try:
        model = _build_detector(monkeypatch, 'VirConv-T.yaml')
        keys_default = list(model.state_dict())
        assert type(model.roi_head).obtain_conf_preds is not part_pool.obtain_conf_preds
    finally:
        _restore_modules(saved)
    monkeypatch.setattr(part_pool, '_reference_obtain_conf_preds', None)
    try:
        model = _build_detector(monkeypatch, 'VirConv-T.yaml', use_fused_part_pool=True)
        head = model.roi_head
        assert type(head).__name__ == 'TEDMHead'
        assert type(head).obtain_conf_preds is part_pool.obtain_conf_preds
        assert part_pool._reference_obtain_conf_preds is not None
        assert part_pool._reference_obtain_conf_preds.__module__ == 'pcdet.models.roi_heads.ted_head'
        assert list(head.grid_offsets) == [0.0, 40.0] and head.featmap_stride == 0.4 and head.num_parts == 49
        assert list(model.state_dict()) == keys_default
    finally:
        _restore_modules(saved)
