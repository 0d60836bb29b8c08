"""Rotated-box IoU / NMS without a GPU: the float64 restatement oracle/iou3d.py against exact convex clipping and against the
outputs of the reference's own kernels (tests/golden/iou3d_ref_*.npz, recorded by oracle/iou3d_golden.py), and the
library's host entry point vc_boxes_iou_bev_host (through iou3d_nms.boxes_bev_iou_cpu and reference_env's
iou3d_nms_cuda.boxes_iou_bev_cpu) against both."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from oracle import iou3d as o
from oracle import iou3d_golden as g

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')
REF = '/root/reference'


def _golden(kind):
    return np.load(os.path.join(GOLDEN, f'iou3d_ref_{kind}.npz'))


def _defined(a, b, three_d=False):
    """pairs with a positive summed area (volume): where both boxes have none, the reference's IoU is the float rounding
    noise of a degenerate polygon divided by the 1e-8 (1e-6) floor — 7.8 for a zero-length box against itself —, not a
    value"""
    va, vb = a[:, 3] * a[:, 4] * (a[:, 5] if three_d else 1), b[:, 3] * b[:, 4] * (b[:, 5] if three_d else 1)
    return va[:, None] + vb[None] > 0


def _clip_area(a, b):
    """exact intersection area of two convex polygons (Sutherland-Hodgman, float64)"""
    poly = o.corners(a)
    clip = o.corners(b)
    for k in range(4):
        c0, c1 = clip[k], clip[(k + 1) % 4]
        side = lambda p: (c1[0] - c0[0]) * (p[1] - c0[1]) - (c1[1] - c0[1]) * (p[0] - c0[0])
        out = []
        for i in range(len(poly)):
            p, q = poly[i], poly[(i + 1) % len(poly)]
            sp, sq = side(p), side(q)
            if sp >= 0:
                out.append(p)
            if (sp >= 0) != (sq >= 0):
                t = sp / (sp - sq)
                out.append((p[0] + t * (q[0] - p[0]), p[1] + t * (q[1] - p[1])))
        poly = out
        if not poly:
            return 0.0
    return abs(sum(poly[i][0] * poly[(i + 1) % len(poly)][1] - poly[(i + 1) % len(poly)][0] * poly[i][1]
                   for i in range(len(poly)))) / 2


def _in_band(box, p):
    """p inside the box with the 1 cm margin but not strictly inside without it"""
    x, y, _, dx, dy, _, h = (float(v) for v in box)
    c, s = np.cos(h), np.sin(h)
    lx, ly = (p[0] - x) * c + (p[1] - y) * s, -(p[0] - x) * s + (p[1] - y) * c
    inside_m = abs(lx) < dx / 2 + o.MARGIN + 1e-6 and abs(ly) < dy / 2 + o.MARGIN + 1e-6
    inside = abs(lx) < dx / 2 - 1e-6 and abs(ly) < dy / 2 - 1e-6
    return inside_m and not inside


def test_oracle_matches_exact_clipping_away_from_the_margin_band():
    boxes = g.cars(400, 7).astype(np.float64)
    n_checked = n_overlap = 0
    for i in range(0, 400, 2):
        for j in range(1, 400, 2):
            a, b = boxes[i], boxes[j]
            if abs(a[0] - b[0]) > 6 or abs(a[1] - b[1]) > 6:
                continue
            if any(_in_band(a, p) for p in o.corners(b)) or any(_in_band(b, p) for p in o.corners(a)):
                continue
            want = _clip_area(a, b)
            assert abs(o.overlap(a, b) - want) <= 1e-9 * max(1.0, want), (i, j)
            n_checked += 1
            n_overlap += want > 0
    assert n_checked > 500 and n_overlap > 200, (n_checked, n_overlap)


def test_oracle_margin_band_counts_a_5mm_gap():
    """rule 2b: boxes 5 mm apart overlap by the band between them (5 mm x the shared edge), not 0"""
    e = g.edge_set().astype(np.float64)
    assert o.overlap(e[0], e[8]) == pytest.approx(0.005 * 2.0, abs=1e-6)
    assert o.overlap(e[0], e[9]) == pytest.approx(0.005 * 4.0, abs=1e-6)
    assert _clip_area(e[0], e[8]) == 0.0


@pytest.mark.parametrize('case', ['rois512_gt48', 'cars300', 'edge'])
def test_oracle_matches_reference_kernel_fixtures(case):
    ref = _golden('iou')
    a, b = g.iou_cases()[case]
    ov = o.matrix(a, b, o.overlap)
    assert np.all(np.abs(ov - ref[case + '_overlap']) <= 2e-5 * np.maximum(1.0, np.abs(ref[case + '_overlap'])))
    ok = _defined(a, b)
    assert np.abs(o.matrix(a, b, o.iou_bev) - ref[case + '_iou_bev'])[ok].max() <= 2e-5
    assert np.abs(o.matrix(a, b, o.iou3d) - ref[case + '_iou3d'])[_defined(a, b, True)].max() <= 2e-5
    assert (ref[case + '_iou_bev'] > 0).sum() >= min(a.shape[0], b.shape[0])


@pytest.mark.parametrize('n', [n for n in g.NMS_SIZES if n <= 65])
def test_oracle_nms_matches_reference_fixtures(n):
    ref = _golden('nms')
    boxes, sc = g.nms_boxes(n)
    for kind in ('rot', 'normal'):
        for thresh in g.NMS_THRESHOLDS:
            idx, keep = ref[f'{kind}_{n}_{thresh}_idx'], ref[f'{kind}_{n}_{thresh}_keep']
            b, s = boxes[idx], sc[idx]
            order = np.argsort(-s, kind='stable')
            got = order[o.nms(b[order], thresh, normal=kind == 'normal')]
            assert np.array_equal(got, keep), (kind, thresh)


@pytest.mark.parametrize('case', ['rois512_gt48', 'cars300', 'edge'])
def test_host_iou_bev_matches_fixtures_and_oracle(lib_built, case):
    from virconv_b200 import iou3d_nms
    from virconv_b200.reference_env import _boxes_iou_bev_cpu
    ref = _golden('iou')[case + '_iou_bev']
    a, b = g.iou_cases()[case]
    got = iou3d_nms.boxes_bev_iou_cpu(a, b)
    assert isinstance(got, np.ndarray) and got.dtype == np.float32
    out = torch.zeros((a.shape[0], b.shape[0]))
    assert _boxes_iou_bev_cpu(torch.from_numpy(a), torch.from_numpy(b), out) == 1
    assert np.array_equal(out.numpy(), got)
    assert np.array_equal(iou3d_nms.boxes_bev_iou_cpu(torch.from_numpy(a), torch.from_numpy(b)).numpy(), got)
    assert np.abs(got - ref)[_defined(a, b)].max() <= 2e-5
    assert np.abs(got - o.matrix(a, b, o.iou_bev)).max() <= 2e-5


def test_nms_over_the_size_limit_is_an_error_code(lib_built):
    from virconv_b200 import _lib
    lib = _lib.load()
    rc = lib.vc_nms_boxes(None, 1, 16385, 7, None, ctypes.c_float(0.5), 0, 10, None, None, None, 0, None)
    assert rc == -4
    assert b'16384' in lib.vc_last_error()
    assert lib.vc_nms_boxes(None, 1, 64, 6, None, ctypes.c_float(0.5), 0, 10, None, None, None, 0, None) == -1
    assert lib.vc_nms_ws_bytes(2, 4000) == 2 * 4000 * 63 * 8


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, 'pcdet')), reason='no /root/reference on this machine')
def test_reference_boxes_bev_iou_cpu_runs_under_reference_env(lib_built):
    """the reference's own iou3d_nms_utils.boxes_bev_iou_cpu, imported unmodified under reference_env.install(), runs on
    the library's host entry point and matches the fixtures"""
    import importlib
    saved = dict(sys.modules)
    try:
        import virconv_b200.reference_env as renv
        renv.install(reference_root=REF)
        utils = importlib.import_module('pcdet.ops.iou3d_nms.iou3d_nms_utils')
        a, b = g.iou_cases()['rois512_gt48']
        got = utils.boxes_bev_iou_cpu(a, b)
        from virconv_b200 import iou3d_nms
        assert np.array_equal(got, iou3d_nms.boxes_bev_iou_cpu(a, b))
        assert np.abs(got - _golden('iou')['rois512_gt48_iou_bev']).max() <= 2e-5
    finally:
        for k in list(sys.modules):
            if k not in saved and k.split('.')[0] in ('pcdet', 'spconv', 'cumm', 'easydict', 'tensorboardX',
                                                      'prefetch_generator', 'skimage'):
                del sys.modules[k]
        for k, v in saved.items():
            sys.modules[k] = v
