"""KITTI evaluation on the H100 (virconv_b200.kitti_eval over csrc/kitti_eval.cu) against what the reference's own
get_official_eval_result recorded (tests/golden/kitti_eval_ref.npz) and against the restatement of oracle/kitti_eval.py
on a 3769-frame synthetic val set."""
import numpy as np
import pytest
import torch

from oracle import kitti_eval as K
from oracle.kitti_eval_golden import CASES
from test_cpu_kitti_eval import case, golden
from virconv_b200 import _lib
from virconv_b200 import kitti_eval as ke

pytestmark = pytest.mark.gpu


def ragged(t, C, K_=2):
    """the thresholds and pr rows in the reference's order (metric, class, difficulty, overlap setting), T rows each"""
    th, pr = [], []
    for m in range(3):
        for c in range(C):
            for d in range(3):
                for k in range(K_):
                    n = t['n_thresholds'][m, c, d, k]
                    th.append(t['thresholds'][m, c, d, k, :n])
                    pr.append(t['pr'][m, c, d, k, :n])
    return np.concatenate(th), np.concatenate(pr)


@pytest.mark.parametrize('name', CASES)
def test_tables_match_reference(name, lib_built):
    z = golden()
    g, d, classes = case(z, name)
    t = ke.eval_tables(g, d, classes, ke._OFFICIAL_MIN_OVERLAPS[:, :, classes], ke._compute_aos(d),
                       return_overlaps=True)
    for m in range(3):
        ref = z[f'{name}.ov{m}']
        got = t['overlaps'][m]
        assert got.shape == ref.shape
        tol = 1e-6 if m != 1 else 2e-6
        assert np.all(np.abs(got - ref) <= tol * np.maximum(np.abs(ref), 1.0)), (m, np.abs(got - ref).max())
    th, pr = ragged(t, len(classes))
    assert np.array_equal(th, z[name + '.th'])
    assert np.array_equal(pr[:, :3], z[name + '.pr'][:, :3])
    np.testing.assert_allclose(pr[:, 3], z[name + '.pr'][:, 3], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize('name', CASES)
def test_official_result_matches_reference(name, lib_built):
    z = golden()
    g, d, classes = case(z, name)
    arg = classes if len(classes) > 1 else ke.CLASS_TO_NAME[classes[0]]
    detail = {}
    s, rd = ke.get_official_eval_result(g, d, arg, PR_detail_dict=detail)
    assert s == str(z[name + '.result_str'])
    assert list(rd) == list(z[name + '.ret_keys'])
    np.testing.assert_allclose(np.array([float(v) for v in rd.values()]), z[name + '.ret_vals'], rtol=0, atol=1e-6)
    for k, v in detail.items():
        np.testing.assert_allclose(v, z[f'{name}.prec_{k}'], rtol=1e-12, atol=0)
    assert sorted(detail) == sorted(k[len(name) + 6:] for k in z.files if k.startswith(name + '.prec_'))


def test_edge_sets(lib_built):
    """no detection anywhere, frames without GT, DontCare-only frames, a class with no GT"""
    g, d = K.synthetic_annos(21, 12, empty=(0, 4))
    for f in (2, 7):
        keep = g[f]['name'] == 'DontCare'
        g[f] = {k: v[keep] for k, v in g[f].items()}
    nod = [{k: v[:0] for k, v in a.items()} for a in d]
    for dets in (d, nod):
        classes = [0, 1, 2, 5]        # no Truck detection is ever made: a class with GT and no match
        mo = np.concatenate([ke._OFFICIAL_MIN_OVERLAPS[:, :, [0, 1, 2]], ke._OFFICIAL_MIN_OVERLAPS[:, :, [5]]], 2)
        aos = ke._compute_aos(dets)
        t = ke.eval_tables(g, dets, classes, mo, aos)
        r = K.evaluate(g, dets, classes, mo, aos)
        for m in range(3):
            np.testing.assert_array_equal(t['precision'][m], r['precision'][m])
            np.testing.assert_array_equal(t['recall'][m], r['recall'][m])
            if aos and m == 0:
                np.testing.assert_allclose(t['orientation'][m], r['orientation'][m], rtol=1e-12)
    s, rd = ke.get_official_eval_result(g, nod, ['Car', 'Cyclist'])
    assert all(v == 0 for v in rd.values()) and 'aos' not in s


def test_bit_identical_and_launch_count(lib_built):
    g, d = K.synthetic_annos(22, 400, check_near=False)
    lib = _lib.load()
    runs = []
    for _ in range(2):
        n0 = lib.vc_launch_count()
        t = ke.eval_tables(g, d, [0, 1, 2], ke._OFFICIAL_MIN_OVERLAPS[:, :, [0, 1, 2]], True, return_overlaps=True)
        assert lib.vc_launch_count() - n0 == 9
        runs.append(t)
    for k in runs[0]:
        assert np.asarray(runs[0][k]).tobytes() == np.asarray(runs[1][k]).tobytes(), k


def test_rotate_iou_eval_against_oracle(lib_built):
    rng = np.random.default_rng(3)
    b = np.c_[rng.uniform(-20, 20, (60, 2)), rng.uniform(0.5, 5, (60, 2)), rng.uniform(-4, 4, 60)]
    q = b[rng.integers(0, 60, 40)] + np.c_[rng.normal(0, 0.5, (40, 2)), np.zeros((40, 2)), rng.normal(0, 0.3, 40)]
    for crit in (-1, 0, 1, 2):
        got = ke.rotate_iou_eval(b, q, crit)
        ref = K.rotate_iou(b, q, crit)
        assert got.dtype == np.float32 and got.shape == (60, 40)
        assert np.all(np.abs(got - ref) <= 2e-6 * np.maximum(np.abs(ref), 1.0)), crit
    assert ke.rotate_iou_eval(b[:0], q).shape == (0, 40)


def test_coco_result_against_oracle(lib_built):
    g, d = K.synthetic_annos(23, 30)
    s = ke.get_coco_eval_result(g, d, ['Car', 'Pedestrian'])
    mo = np.zeros((10, 3, 2))
    mo[:, :, 0] = np.linspace(0.5, 0.95, 10)[:, None]
    mo[:, :, 1] = np.linspace(0.25, 0.7, 10)[:, None]
    r = K.evaluate(g, d, [0, 1], mo, True)
    ap = ke.get_mAP(r['precision'][2]).mean(-1)
    lines = s.splitlines()
    assert lines[0] == 'Car coco AP@0.50:0.05:0.95:' and lines[5] == 'Pedestrian coco AP@0.25:0.05:0.70:'
    assert lines[3] == f'3d   AP:{ap[0, 0]:.2f}, {ap[0, 1]:.2f}, {ap[0, 2]:.2f}'


def test_val_set_against_oracle(lib_built):
    """a 3769-frame synthetic val set (KITTI val's size), Car / Pedestrian / Cyclist"""
    g, d = K.synthetic_annos(24, 3769)
    classes = [0, 1, 2]
    mo = ke._OFFICIAL_MIN_OVERLAPS[:, :, classes]
    t = ke.eval_tables(g, d, classes, mo, True, return_overlaps=True)
    r = K.evaluate(g, d, classes, mo, True)
    for m in range(3):
        ref = np.concatenate([o.ravel() for o in r['overlaps'][m]])
        assert np.all(np.abs(t['overlaps'][m] - ref) <= 2e-6 * np.maximum(np.abs(ref), 1.0)), m
        for c in range(3):
            for dd in range(3):
                for k in range(2):
                    n = t['n_thresholds'][m, c, dd, k]
                    assert np.array_equal(t['thresholds'][m, c, dd, k, :n], r['thresholds'][m][(c, dd, k)])
                    assert np.array_equal(t['pr'][m, c, dd, k, :n, :3], r['pr'][m][(c, dd, k)][:, :3])
        np.testing.assert_allclose(t['precision'][m], r['precision'][m], rtol=1e-12, atol=0)
    np.testing.assert_allclose(t['orientation'][0], r['orientation'][0], rtol=1e-9, atol=0)
    assert torch.cuda.is_available()
