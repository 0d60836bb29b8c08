"""RPN anchor mask and target assignment without a GPU: the float32 restatement oracle/anchor_targets.py against the
reference's own `AnchorHeadSingle.get_anchor_mask` and `AxisAlignedTargetAssigner.assign_targets`
(tests/golden/anchor_targets_ref.npz, recorded by oracle/anchor_targets_golden.py), the wrap and trimming rules on
hand-built cases, the library's new symbols, the constructor's limits, and — where the reference's sources exist — the
VirConv-L detector built with `reference_env.install(use_fused_rpn_targets=True)`."""
import os
import sys

import numpy as np
import pytest

from oracle import anchor_targets as o
from oracle import anchor_targets_golden as g
from test_cpu_voxel_pool import _build_virconv_l, _restore_modules, need_ref

SYMS = ('vc_anchor_mask', 'vc_anchor_targets_ws_bytes', 'vc_anchor_targets')


def golden():
    return np.load(os.path.join(os.path.dirname(__file__), 'golden', 'anchor_targets_ref.npz'))


def case_inputs(z, case):
    """(ordered anchors [N, 7], set index [N], gt, class names, anchor class names, matched, unmatched) of a golden case"""
    sets = [g.CAR] if case == 'L' else g.SETS_T
    m = z[f'{case}.mask']
    per_set = [o.anchors_from_shifts(z[f'{case}.x_shifts{s}'], z[f'{case}.y_shifts{s}'], c['anchor_bottom_heights'],
                                     c['anchor_sizes'], c['anchor_rotations'])[:, m] for s, c in enumerate(sets)]
    anchors, sid = o.ordered(per_set)
    names = g.CLASS_NAMES_L if case == 'L' else g.CLASS_NAMES_T
    return (anchors, sid, z[f'{case}.gt'], names, [c['class_name'] for c in sets], [c['matched_threshold'] for c in sets],
            [c['unmatched_threshold'] for c in sets])


def mask_args(shape=g.FEATURE_SHAPE_L):
    from virconv_b200.anchor_targets import mask_params
    return (*mask_params(g.PCR, g.GRID), shape[-2], shape[-1])


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def test_oracle_mask_matches_reference():
    z = golden()
    assert np.array_equal(o.anchor_mask(z['L.points'], *mask_args()), z['L.mask'])


@pytest.mark.parametrize('case', ['L', 'T'])
def test_oracle_targets_match_reference(case):
    z = golden()
    labels, targets, reg, ious = o.assign(*case_inputs(z, case))
    assert np.array_equal(labels, z[f'{case}.box_cls_labels'])
    assert np.array_equal(bits(ious), bits(z[f'{case}.gt_ious']))          # incl. the sign of -0.0
    assert np.array_equal(reg, z[f'{case}.reg_weights'])
    assert np.abs(targets - z[f'{case}.box_reg_targets']).max() <= 1e-6


def test_golden_covers_edge_cases():
    z = golden()
    m = z['L.mask']
    assert 0.1 < m.mean() < 0.9
    assert m[190:200].any() and m[:, 170:176].any()                          # set only through the fine wrap
    anchors, sid, gt, *_ = case_inputs(z, 'L')
    n0 = o.trimmed_count(gt[0])
    assert n0 < g.M_GT and (gt[0, :n0, :7].sum(1) == 0).any()                 # ragged, with an interior zero row
    assert (gt[0, :n0, 7] == 0).any()
    assert not gt[1].any() and o.trimmed_count(gt[1]) == 1
    assert (bits(z['L.gt_ious'][1]) == 0).all()                               # the kept zero row: +0.0, not -0.0
    u, c = np.unique(gt[0, :n0], axis=0, return_counts=True)
    assert (c[u[:, 3] > 0] > 1).any()                                         # a duplicated box
    iou = o.iou_nearest(anchors, gt[0, :n0, :7])
    col = iou.max(0)
    assert ((iou == col[None]) & (col[None] > 0)).sum(0).max() >= 2           # tied column maxima
    r = np.abs(o.nearest_bev(gt[0, :n0])[0][:, 2] - o.nearest_bev(gt[0, :n0])[0][:, 0] - gt[0, :n0, 3]) > 1e-3
    assert r.any() and (~r[gt[0, :n0, 3] > 0]).any()                          # headings on both sides of the swap
    lab = z['L.box_cls_labels'][0]
    assert (lab > 0).sum() > 10 and (lab < 0).any()
    # case T: interleaved sets, one scene without cyclists
    anchors, sid, gt, *_ = case_inputs(z, 'T')
    assert list(sid[:6]) == [0, 0, 1, 1, 2, 2]
    assert (bits(z['T.gt_ious'][1][sid == 2]) == 0x80000000).all()
    for s in range(3):
        assert (z['T.box_cls_labels'][0][sid == s] > 0).any()


def test_mask_wrap_rules():
    args = mask_args()
    m = o.anchor_mask(np.array([[0, 1.0, -39.0]], np.float32), *args)     # coarse (0, 0)
    rows, cols = np.nonzero(m.any(1))[0], np.nonzero(m.any(0))[0]
    assert list(rows) == list(range(0, 10)) + list(range(190, 200))
    assert list(cols) == list(range(0, 10)) + list(range(166, 176))
    m = o.anchor_mask(np.array([[0, -5.0, 1.0]], np.float32), *args)      # x / 4 = -1.25 -> -1 -> coarse column 16
    assert list(np.nonzero(m.any(0))[0]) == list(range(150, 170))
    m = o.anchor_mask(np.array([[0, 500.0, 500.0]], np.float32), *args)   # clamped from above to the last coarse cell
    assert list(np.nonzero(m.any(1))[0]) == list(range(180, 200))
    assert list(np.nonzero(m.any(0))[0]) == list(range(150, 170))
    assert not o.anchor_mask(np.zeros((0, 3), np.float32), *args).any()


def test_trimming_rules():
    gt = np.zeros((5, 8), np.float32)
    assert o.trimmed_count(gt) == 1                                           # row 0 always stays
    gt[1, 0] = 1
    assert o.trimmed_count(gt) == 2
    gt[3, 7] = 1                                                              # a class but a zero box: trimmed
    assert o.trimmed_count(gt) == 2
    gt[3, 3] = 2                                                              # interior zero row 2 stays
    assert o.trimmed_count(gt) == 4
    assert o.trimmed_count(np.zeros((0, 8), np.float32)) == 0


def test_class_names_wrap():
    from virconv_b200.anchor_targets import name_sets
    assert name_sets(['Car', 'Pedestrian', 'Cyclist'], ['Car', 'Pedestrian', 'Cyclist']) == [1, 2, 4]
    assert name_sets(['Car', 'Van'], ['Car']) == [1, 0]
    a = np.array([[10.0, 0.0, 0.0, 3.9, 1.6, 1.5, 0.0]], np.float32)
    gt = np.array([[[10.0, 0.0, 0.0, 3.9, 1.6, 1.5, 0.0, 0.0]]], np.float32)      # class 0 -> class_names[-1]
    lab = o.assign(a, np.zeros(1, np.int32), gt, ['Car', 'Cyclist'], ['Cyclist'], [0.6], [0.45])[0]
    assert lab[0, 0] == 0                                                     # matched, but its label is the class 0
    lab, _, _, ious = o.assign(a, np.zeros(1, np.int32), gt, ['Car', 'Cyclist'], ['Car'], [0.6], [0.45])
    assert lab[0, 0] == 0 and bits(ious)[0, 0] == 0x80000000                  # no GT for the set


def test_new_symbols_exported():
    from virconv_b200 import _lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include',
                               'virconv_b200.h')).read()
    for sym in SYMS:
        assert sym in _lib.SIGNATURES
        assert f' {sym}(' in header


def test_library_exports_new_symbols(lib_built):
    import ctypes
    lib = ctypes.CDLL(lib_built)
    for sym in SYMS:
        assert hasattr(lib, sym)


def test_constructor_rejects_what_is_not_compiled_in():
    from virconv_b200.anchor_targets import AxisAlignedTargetAssigner
    from virconv_b200.reference_env import EasyDict

    class Coder:
        code_size = 7
    AxisAlignedTargetAssigner(g.model_cfg([g.CAR]), ['Car'], Coder(), g.GRID, g.PCR)
    bad = [dict(), dict(), dict(), dict()]
    bad[0]['model_cfg'] = EasyDict(g.model_cfg([g.CAR]), USE_MULTIHEAD=True)
    bad[1]['match_height'] = True
    cfg = g.model_cfg([g.CAR])
    cfg.TARGET_ASSIGNER_CONFIG.POS_FRACTION = 0.5
    bad[2]['model_cfg'] = cfg
    coder = Coder()
    coder.code_size = 8
    bad[3]['box_coder'] = coder
    for kw in bad:
        args = dict(model_cfg=g.model_cfg([g.CAR]), class_names=['Car'], box_coder=Coder(), grid_size=g.GRID,
                    point_cloud_range=g.PCR)
        args.update(kw)
        with pytest.raises(ValueError, match='reference class'):
            AxisAlignedTargetAssigner(**args)


@need_ref
def test_virconv_l_head_uses_fused_assigner(monkeypatch):
    from virconv_b200 import anchor_targets
    saved = dict(sys.modules)
    try:
        keys_default = list(_build_virconv_l(monkeypatch).state_dict())
    finally:
        _restore_modules(saved)
    try:
        model = _build_virconv_l(monkeypatch, use_fused_rpn_targets=True)
        head = model.dense_head
        assert type(head.target_assigner) is anchor_targets.AxisAlignedTargetAssigner
        assert type(head).get_anchor_mask is anchor_targets.get_anchor_mask
        assert head.target_assigner._matched == [0.6] and head.target_assigner._name_sets == [1]
        assert list(model.state_dict()) == keys_default
    finally:
        _restore_modules(saved)
