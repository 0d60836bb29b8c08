"""Box decoding and cascade stage transforms without a GPU: the restatements of oracle/box_decode.py against the reference's
own `generate_predicted_boxes` (anchor and RoI heads) and `TEDMHead.roi_x_trans / roi_score_trans / pred_x_trans`
(tests/golden/box_decode_ref.npz, recorded by oracle/box_decode_golden.py), the coverage of the golden cases, the
library's new symbols and argument checks, the Python operators' device checks, refusals and fallbacks, and — where the
reference's sources exist — the VirConv-T detector built with `reference_env.install(use_fused_box_decode=True)`."""
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import box_decode as o
from oracle import box_decode_golden as g
from test_cpu_part_pool import _build_detector
from test_cpu_voxel_pool import _restore_modules, need_ref

SYMS = ('vc_anchor_decode', 'vc_anchor_decode_bwd', 'vc_roi_decode', 'vc_roi_decode_bwd', 'vc_box_xtrans')
RPN = ('A1', 'A2', 'A3')
RCNN = ('R1', 'R50', 'R160')
PERIOD = 2 * np.pi / g.NUM_DIR_BINS


def golden():
    return g.load(os.path.join(os.path.dirname(__file__), 'golden', 'box_decode_ref.npz'))


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def ulp_tol(ref, ulps):
    """`ulps` ulp of the largest magnitude, per column"""
    r = np.asarray(ref, np.float32).reshape(-1, ref.shape[-1])
    return ulps * np.spacing(np.abs(r).max(0)).astype(np.float64)


def within(got, ref, ulps):
    err = np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64)).reshape(-1, ref.shape[-1])
    return bool((err <= ulp_tol(ref, ulps)).all())


def rpn_args(z, case):
    return (z[f'{case}.box'], g.rpn_anchors(z, case), z[f'{case}.dir'] if f'{case}.dir' in z else None,
            g.DIR_OFFSET, g.DIR_LIMIT_OFFSET, PERIOD)


@pytest.mark.parametrize('case', RPN)
def test_oracle_matches_reference_rpn(case):
    z = golden()
    args = rpn_args(z, case)
    assert rel(o.anchor_decode(*args), z[f'{case}.out']) < 1e-12
    got = o.anchor_decode(*args, dtype=np.float32, div=True)
    ref = z[f'f32.{case}.out']
    assert within(got[..., :6], ref[..., :6], 2)
    # the heading: the same float32 operations as torch's CPU kernels, its division by the period a true division
    assert np.array_equal(got[..., 6], ref[..., 6])
    if f'{case}.g' in z:
        d = o.anchor_decode_grad(z[f'{case}.g'], args[0], args[1])
        assert rel(d, z[f'{case}.dbox']) < 1e-12
        assert within(o.anchor_decode_grad(z[f'{case}.g'], args[0], args[1], np.float32), z[f'f32.{case}.dbox'], 2)


@pytest.mark.parametrize('case', RCNN)
def test_oracle_matches_reference_rcnn(case):
    z = golden()
    box, rois, gr = z[f'{case}.box'], z[f'{case}.rois'], z[f'{case}.g']
    assert rel(o.roi_decode(box, rois), z[f'{case}.out']) < 1e-12
    assert within(o.roi_decode(box, rois, np.float32), z[f'f32.{case}.out'], 2)
    assert rel(o.roi_decode_grad(gr, box, rois), z[f'{case}.dbox']) < 1e-12
    assert within(o.roi_decode_grad(gr, box, rois, np.float32), z[f'f32.{case}.dbox'], 2)


STAGES = {'roi_x_trans': lambda i: (i - 1, i), 'roi_score_trans': lambda i: (i, 0), 'pred_x_trans': lambda i: (i, None)}


@pytest.mark.parametrize('method', g.XT_METHODS)
def test_oracle_matches_reference_xtrans(method):
    z = golden()
    boxes, tp = z['X.boxes'], z['X.tparam']
    for R in (1, 2, 3):
        for i in range(3):
            frm, to = STAGES[method](o.clamp_stage(i, R))
            key = f'X.{method}.{R}.{g.clamp(i, R)}'
            assert rel(o.xtrans(boxes, tp[:, :R], frm, to), z[key]) < 1e-12, key
            got = o.xtrans(boxes, tp[:, :R], frm, to, np.float32)
            assert within(got, z[f'f32.{key}'], 2), key
            assert np.array_equal(got[..., 3:], z[f'f32.{key}'][..., 3:]), key     # sizes, heading, extra columns


def test_golden_bin_edges_are_unambiguous():
    """every golden heading that lies within a few ulp of a limit_period bin edge has the same bin under torch's CPU
    division and its CUDA reciprocal multiplication, so the kernel must reproduce it; `amb` records exactly that"""
    z = golden()
    near = 0
    for case in ('A1', 'A2'):
        h = z[f'{case}.box'][..., 6] + g.rpn_anchors(z, case)[None, :, 6]
        assert np.array_equal(z[f'{case}.amb'], g.ambiguous(h))
        assert not z[f'{case}.amb'].any()
        q = o.bin_quotient(np.float32(h) - np.float32(g.DIR_OFFSET), PERIOD, g.DIR_LIMIT_OFFSET, np.float32)
        edge = np.abs(q - np.round(q)) <= 8 * np.spacing(np.maximum(np.abs(q), np.float32(1)))
        near += int(edge.sum())
        assert (q[edge] == np.round(q[edge])).any() and (q[edge] < np.round(q[edge])).any()   # on and below an edge
    assert near >= 2 * 27


def test_golden_covers_edge_cases():
    z = golden()
    assert z['A1.box'].shape == (1, 70400, 7) and z['anchors'].shape == (70400, 7)
    assert z['A2.box'].shape[0] == 2 and z['A2.box'].shape[1] < 70400 and 'A3.dir' not in z
    assert {z[f'{c}.rois'].shape[:2] for c in RCNN} == {(1, 1), (2, 50), (2, 160)}
    assert z['R50.rois'].shape[2] == 9 and z['X.boxes'].shape[2] == 9                     # extra columns
    rois = z['R160.rois'].reshape(-1, 7)
    for h in (0.0, np.pi / 2, -np.pi / 2, np.pi):
        assert (rois[:, 6] == np.float32(h)).any() and (z['X.boxes'][..., 6] == np.float32(h)).any()
        assert (z['A1.box'][..., 6] == np.float32(h)).any()
    assert (np.abs(rois[:, 3:6]).sum(1) == 0).any()                                         # zero-size RoIs
    for c in ('A1', 'A2'):
        d = z[f'{c}.dir']
        assert (d[..., 0] == d[..., 1]).sum() >= 8                                          # tied logits
    assert np.array_equal(z['X.tparam'][0], np.float32(g.XT_VIRCONV_T))
    assert {k.split('.')[2] for k in z if k.startswith('X.roi_x_trans.')} == {'1', '2', '3'}


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
    assert lib.vc_anchor_decode(p, p, p, -1, 10, 2, 0.0, 0.0, 3.14, p, None) == -1
    assert lib.vc_anchor_decode(p, p, p, 2, 10, 0, 0.0, 0.0, 3.14, p, None) == -1       # a classifier without bins
    assert lib.vc_anchor_decode(p, None, p, 2, 0, 0, 0.0, 0.0, 3.14, p, None) == 0      # no anchor: nothing to do
    assert lib.vc_roi_decode(p, p, 2, 10, 6, p, None) == -1                             # a RoI row shorter than 7
    assert lib.vc_roi_decode_bwd(p, p, p, 2, 0, 7, p, None) == 0
    assert lib.vc_box_xtrans(p, p, 2, 10, 7, 0, -1, -1, p, None) == -1                  # no stage
    assert lib.vc_box_xtrans(p, p, 2, 10, 7, 3, 3, 0, p, None) == -1                    # a stage beyond R
    assert lib.vc_box_xtrans(p, p, 2, 0, 7, 3, 0, 1, p, None) == 0


def _anchor_head(**kw):
    from virconv_b200 import box_decode
    coder = type('ResidualCoder', (), {'code_size': 7, 'encode_angle_by_sincos': False})()
    head = types.SimpleNamespace(anchors=[torch.zeros(1, 4, 1, 2, 7)], use_multihead=False, box_coder=coder,
                                 model_cfg=types.SimpleNamespace(DIR_OFFSET=0.78539, DIR_LIMIT_OFFSET=0.0,
                                                                 NUM_DIR_BINS=2))
    for k, v in kw.items():
        setattr(head, k, v)
    return head, box_decode


def test_operators_reject_cpu_tensors():
    from virconv_b200._lib import VirConvLibraryError
    from virconv_b200.box_decode import anchor_decode, box_xtrans, roi_decode
    with pytest.raises(VirConvLibraryError):
        anchor_decode(torch.zeros(1, 8, 7), torch.zeros(8, 7))
    with pytest.raises(VirConvLibraryError):
        roi_decode(torch.zeros(3, 7), torch.zeros(1, 3, 7))
    with pytest.raises(VirConvLibraryError):
        box_xtrans(torch.zeros(1, 3, 7), torch.zeros(1, 3, 3), 0, 1)
    head, bd = _anchor_head()
    with pytest.raises(VirConvLibraryError):
        bd.anchor_generate_predicted_boxes(head, 1, torch.zeros(1, 4, 2), torch.zeros(1, 4, 14), torch.zeros(1, 4, 4))


def test_unsupported_configurations_name_the_reference():
    head, bd = _anchor_head()
    cls, box, dirs = torch.zeros(1, 4, 2), torch.zeros(1, 4, 14), torch.zeros(1, 4, 4)
    prev = type('PreviousResidualDecoder', (), {'code_size': 7})()
    sincos = type('ResidualCoder', (), {'code_size': 8, 'encode_angle_by_sincos': True})()
    bad = [(dict(box_coder=prev), (cls, box, dirs)), (dict(box_coder=sincos), (cls, box, dirs)),
           (dict(use_multihead=True), (cls, box, dirs)), ({}, (cls, [box], dirs)), ({}, (cls, box.double(), dirs))]
    for attrs, args in bad:
        h, _ = _anchor_head(**attrs)
        with pytest.raises(ValueError, match='AnchorHeadTemplate.generate_predicted_boxes'):
            bd.anchor_generate_predicted_boxes(h, 1, *args)
    rhead = types.SimpleNamespace(box_coder=sincos)
    with pytest.raises(ValueError, match='RoIHeadTemplate.generate_predicted_boxes'):
        bd.roi_generate_predicted_boxes(rhead, 1, torch.zeros(1, 3, 7), torch.zeros(3, 1), torch.zeros(3, 8))
    xhead = types.SimpleNamespace(x_trans_train=types.SimpleNamespace(aug_config_list=[{'NAME': 'world_scaling'}]))
    with pytest.raises(ValueError, match='TEDMHead.pred_x_trans'):
        bd.pred_x_trans(xhead, torch.zeros(1, 3, 7), 0, torch.zeros(1, 3, 3))


def test_gradient_inputs_go_to_reference_methods(monkeypatch):
    from virconv_b200 import box_decode as bd
    head = types.SimpleNamespace()
    rois = torch.zeros(1, 3, 7, requires_grad=True)
    monkeypatch.setattr(bd, '_reference_roi_generate_predicted_boxes', None)
    with pytest.raises(RuntimeError, match='reference method'):
        bd.roi_generate_predicted_boxes(head, 1, rois, torch.zeros(3, 1), torch.zeros(3, 7))
    calls = []
    monkeypatch.setattr(bd, '_reference_roi_generate_predicted_boxes', lambda *a: calls.append(a) or 'ref')
    assert bd.roi_generate_predicted_boxes(head, 1, rois, torch.zeros(3, 1), torch.zeros(3, 7)) == 'ref'
    assert calls[0][0] is head and calls[0][2] is rois
    tp = torch.zeros(1, 3, 3)
    for name in g.XT_METHODS:
        monkeypatch.setattr(bd, f'_reference_{name}', None)
        with pytest.raises(RuntimeError, match='reference method'):
            getattr(bd, name)(head, rois, 1, tp)
        calls = []
        monkeypatch.setattr(bd, f'_reference_{name}', lambda *a: calls.append(a) or name)
        assert getattr(bd, name)(head, rois, 1, tp) == name
        assert calls[0][0] is head and calls[0][1] is rois and calls[0][2] == 1 and calls[0][3] is tp


@need_ref
def test_virconv_t_heads_use_fused_box_decode(monkeypatch):
    from virconv_b200 import box_decode as bd
    saved = dict(sys.modules)
    names = ('_reference_anchor_generate_predicted_boxes', '_reference_roi_generate_predicted_boxes',
             '_reference_roi_x_trans', '_reference_roi_score_trans', '_reference_pred_x_trans')
    try:
        model = _build_detector(monkeypatch, 'VirConv-T.yaml')
        keys_default = list(model.state_dict())
        assert type(model.roi_head).roi_x_trans is not bd.roi_x_trans
    finally:
        _restore_modules(saved)
    for n in names:
        monkeypatch.setattr(bd, n, None)
    try:
        model = _build_detector(monkeypatch, 'VirConv-T.yaml', use_fused_box_decode=True)
        rpn, head = model.dense_head, model.roi_head
        assert type(head).__name__ == 'TEDMHead'
        assert type(rpn).generate_predicted_boxes is bd.anchor_generate_predicted_boxes
        assert type(head).generate_predicted_boxes is bd.roi_generate_predicted_boxes
        for m in g.XT_METHODS:
            assert getattr(type(head), m) is getattr(bd, m)
        modules = ('pcdet.models.dense_heads.anchor_head_template', 'pcdet.models.roi_heads.roi_head_template',
                   'pcdet.models.roi_heads.ted_head', 'pcdet.models.roi_heads.ted_head', 'pcdet.models.roi_heads.ted_head')
        for n, mod in zip(names, modules):
            assert getattr(bd, n) is not None and getattr(bd, n).__module__ == mod, n
        assert tuple(c['NAME'] for c in head.x_trans_train.aug_config_list) == bd.XTRANS_ORDER
        assert type(rpn.box_coder).__name__ == 'ResidualCoder' and rpn.box_coder.code_size == 7
        assert list(model.state_dict()) == keys_default
    finally:
        _restore_modules(saved)
