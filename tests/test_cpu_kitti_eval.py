"""KITTI evaluation without a GPU: the restatement of oracle/kitti_eval.py against what the reference's own
get_official_eval_result recorded (tests/golden/kitti_eval_ref.npz), the host packing and argument checks of
virconv_b200.kitti_eval, and — where the reference's sources exist — the binding of reference_env.install(
use_fused_kitti_eval=True)."""
import ctypes
import importlib
import sys

import numpy as np
import pytest

from oracle import kitti_eval as K
from oracle.kitti_eval_golden import CASES, unpack_annos
from test_cpu_voxel_pool import REF, _restore_modules, need_ref
from virconv_b200 import kitti_eval as ke

GOLDEN = 'tests/golden/kitti_eval_ref.npz'


def golden():
    import os
    return np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), GOLDEN))


def case(z, name):
    g, d = unpack_annos(name + '.gt', z), unpack_annos(name + '.dt', z)
    classes = [int(c) if c.isdigit() else ke._class_ids(str(c), ke.CLASS_TO_NAME)[0] for c in z[name + '.classes']]
    return g, d, classes


def flat_tables(r, C, K_=2):
    keys = [(m, c, d, k) for m in range(3) for c in range(C) for d in range(3) for k in range(K_)]
    th = np.concatenate([r['thresholds'][m][(c, d, k)] for m, c, d, k in keys])
    pr = np.concatenate([r['pr'][m][(c, d, k)] for m, c, d, k in keys])
    return th, pr


@pytest.mark.parametrize('name', CASES)
def test_oracle_matches_reference(name):
    z = golden()
    g, d, classes = case(z, name)
    r = K.evaluate(g, d, classes, ke._OFFICIAL_MIN_OVERLAPS[:, :, classes], ke._compute_aos(d))
    for m in range(3):
        ov = np.concatenate([o.ravel() for o in r['overlaps'][m]]) if r['overlaps'][m] else np.zeros(0)
        ref = z[f'{name}.ov{m}']
        assert ov.shape == ref.shape
        if m == 0:
            assert np.array_equal(ov, ref)
        else:   # float32 rounding of the rotated-box geometry: within 2 ulp
            assert np.all(np.abs(ov - ref) <= 2.5e-7 * np.maximum(np.abs(ref), 1.0)), np.abs(ov - ref).max()
    th, pr = flat_tables(r, len(classes))
    assert np.array_equal(th, z[name + '.th'])
    assert np.array_equal(pr[:, :3], z[name + '.pr'][:, :3])
    np.testing.assert_allclose(pr[:, 3], z[name + '.pr'][:, 3], rtol=1e-12, atol=1e-12)
    for key, m in (('bbox', 0), ('bev', 1), ('3d', 2)):
        np.testing.assert_allclose(r['precision'][m], z[f'{name}.prec_{key}'], rtol=1e-12, atol=0)
    if name + '.prec_aos' in z.files:
        np.testing.assert_allclose(r['orientation'][0], z[name + '.prec_aos'], rtol=1e-12, atol=0)


def test_golden_pins_the_edge_cases():
    """what the reference returns on the edge cases, as recorded"""
    z = golden()
    # no detection anywhere: no AOS line, no threshold, every AP 0
    assert np.all(z['nodet.th_n'] == 0) and 'aos' not in str(z['nodet.result_str'])
    assert np.all(z['nodet.ret_vals'] == 0)
    # the edge case has no Cyclist GT: its thresholds are empty and its APs 0
    keys = list(z['edge.ret_keys'])
    assert all(z['edge.ret_vals'][keys.index(k)] == 0 for k in keys if k.startswith('Cyclist'))
    g, d, _ = case(z, 'edge')
    assert [len(a['name']) for a in g][0] == 0 and all(n == 'DontCare' for n in g[2]['name'])
    # detections with alpha -10: no AOS
    assert 'aos' not in str(z['noaos.result_str']) and not any('aos' in k for k in z['noaos.ret_keys'])


def test_golden_keeps_clear_of_min_overlaps():
    """no recorded overlap lies within oracle.kitti_eval.NEAR of a min-overlap value"""
    z = golden()
    vals = np.concatenate([z[f'{n}.ov{m}'] for n in CASES for m in range(3)])
    assert np.min(np.abs(vals[:, None] - np.array(K.MIN_OVERLAP_VALUES)[None, :])) >= K.NEAR


def test_pack_layout():
    g, d = K.synthetic_annos(5, 6, check_near=False, empty=(2,))
    gt, dt, offs, P = ke.pack(g, d)
    ng, nd = [len(a['name']) for a in g], [len(a['name']) for a in d]
    assert gt.shape == (sum(ng), ke.ROW) and dt.shape == (sum(nd), ke.ROW)
    assert list(np.diff(offs[0])) == ng and list(np.diff(offs[1])) == nd
    assert list(np.diff(offs[2])) == [a * b for a, b in zip(ng, nd)] and P == offs[2, -1]
    r = 0
    for a in g:
        for i, n in enumerate(a['name']):
            row = gt[r]
            assert np.array_equal(row[:4], a['bbox'][i]) and row[4] == a['alpha'][i]
            assert np.array_equal(row[5:8], a['location'][i]) and np.array_equal(row[8:11], a['dimensions'][i])
            assert row[11] == a['rotation_y'][i] and row[12] == a['truncated'][i] and row[13] == a['occluded'][i]
            assert row[14] == {'car': 0, 'pedestrian': 1, 'cyclist': 2, 'van': 3, 'person_sitting': 4,
                               'truck': 5}.get(n.lower(), -1)
            assert row[15] == (n == 'DontCare')
            r += 1
    r = 0
    for a in d:
        for j in range(len(a['name'])):
            assert dt[r, 12] == np.float64(a['score'][j]) and dt[r, 4] == a['alpha'][j]
            r += 1


def test_argument_checks():
    g, d = K.synthetic_annos(5, 3, check_near=False)
    with pytest.raises(ValueError, match='frames'):
        ke.pack(g, d[:2])
    bad = [dict(a) for a in d]
    bad[1]['bbox'] = bad[1]['bbox'][:, :3]
    with pytest.raises(ValueError, match='bbox'):
        ke.pack(g, bad)
    with pytest.raises(ValueError, match='classes'):
        ke.eval_tables(g, d, [7], np.zeros((2, 3, 1)), False)
    with pytest.raises(ValueError, match='min_overlaps'):
        ke.eval_tables(g, d, [0], np.zeros((2, 2, 1)), False)
    with pytest.raises(ValueError, match='metric'):
        ke.eval_overlaps(g, d, 3)
    with pytest.raises(KeyError):
        ke.get_official_eval_result(g, d, ['Tram'])
    assert ke._class_ids('Car', ke.CLASS_TO_NAME) == [0] and ke._class_ids(['Pedestrian', 2], ke.CLASS_TO_NAME) == [1, 2]


def test_library_limits(lib_built):
    """arguments the C entry points refuse before they enqueue anything"""
    from virconv_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(16)   # never dereferenced: every call below returns before a launch
    assert lib.vc_kitti_overlaps(p, p, p, 2, 10, 3, p, None) == -1            # no metric 3
    assert lib.vc_kitti_overlaps(p, p, p, 2, 0, 1, p, None) == 0              # no pair: nothing to do
    assert lib.vc_kitti_rotate_iou(p, p, -1, 2, -1, p, None) == -1
    assert lib.vc_kitti_rotate_iou(p, p, 0, 2, -1, p, None) == 0
    assert lib.vc_kitti_eval_ws_bytes(10, 20, 20, 0, 2) == 0
    ws = lib.vc_kitti_eval_ws_bytes(10, 20, 20, 3, 2)
    assert ws > 0
    cls = _lib.host_i32([0, 1, 2])
    assert lib.vc_kitti_eval(p, p, p, p, 10, 20, 20, 40, 3, cls, 11, 0, p, p, p, ws, None) == -1   # K > 10
    assert lib.vc_kitti_eval(p, p, p, p, 10, 20, 20, 40, 3, _lib.host_i32([0, 1, 6]), 2, 0, p, p, p, ws, None) == -1
    assert lib.vc_kitti_eval(p, p, p, p, 10, 20, 20, 40, 3, cls, 2, 0, p, p, p, ws - 1, None) == -1  # workspace


@need_ref
def test_reference_env_binds_fused_eval():
    saved = dict(sys.modules)
    try:
        from virconv_b200 import reference_env
        reference_env.install(reference_root=REF, use_fused_kitti_eval=True)
        ev = importlib.import_module('pcdet.datasets.kitti.kitti_object_eval_python.eval')
        assert ev.get_official_eval_result is ke.get_official_eval_result
        assert ev.get_coco_eval_result is ke.get_coco_eval_result
        assert ev.rotate_iou_gpu_eval is ke.rotate_iou_eval
        # KittiDatasetMM.evaluation imports the module inside the method and calls the function through it
        ds = importlib.import_module('pcdet.datasets.kitti.kitti_dataset_mm')
        calls = []
        orig = ke.get_official_eval_result
        ev.get_official_eval_result = lambda gt, dt, names: calls.append((gt, dt, names)) or ('s', {'k': 1})
        try:
            self = type('S', (), {'kitti_infos': [{'annos': {'name': np.array(['Car'])}}]})()
            out = ds.KittiDatasetMM.evaluation(self, [{'name': np.array(['Car'])}], ['Car'])
        finally:
            ev.get_official_eval_result = orig
        assert out == ('s', {'k': 1}) and calls and calls[0][2] == ['Car']
        # and the name it resolves is the fused function
        src = importlib.import_module('inspect').getsource(ds.KittiDatasetMM.evaluation)
        assert 'kitti_eval.get_official_eval_result' in src
        assert importlib.import_module('pcdet.datasets.kitti.kitti_object_eval_python').eval.get_official_eval_result \
            is ke.get_official_eval_result
    finally:
        _restore_modules(saved)
