"""Detection losses without a GPU: the float64 restatement oracle/head_losses.py (losses and closed-form gradients)
against the reference's own `AnchorHeadTemplate.get_loss` / `RoIHeadTemplate.get_loss` and their autograd gradients
(tests/golden/head_losses_ref.npz, recorded by oracle/head_losses_golden.py), the edge cases the fixture holds, the
configuration checks, the library's new symbols, the anchor order, and — where the reference's sources exist — the
VirConv-L detector built with `reference_env.install(use_fused_losses=True)`."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import head_losses as o
from oracle import head_losses_golden as g
from test_cpu_voxel_pool import _build_virconv_l, _restore_modules, need_ref

SYMS = ('vc_rpn_loss_ws_bytes', 'vc_rpn_loss', 'vc_rcnn_loss_ws_bytes', 'vc_rcnn_loss')
RPN_CASES = {'L': 1, 'C3': 3}
RCNN_CASES = ('R1', 'R3', 'T')


def golden():
    return np.load(os.path.join(os.path.dirname(__file__), 'golden', 'head_losses_ref.npz'))


def rel(a, b):
    """max |a - b| over max |b|"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def rpn_inputs(z, case):
    return tuple(z[f'{case}.{k}'] for k in ('cls_preds', 'box_preds', 'dir_cls_preds', 'box_cls_labels',
                                             'box_reg_targets', 'anchors_flat'))


def rcnn_branches(z, case):
    """[(dict of numpy arrays, weight), ...] in the reference's order, and the branch names"""
    order = g.branch_order(list(z[f'{case}.branches']))
    return [({k: z[f'{case}.{b}.{k}'] for k in g.RCNN_KEYS}, w) for b, w in order], [b for b, _ in order]


@pytest.mark.parametrize('case', list(RPN_CASES))
def test_rpn_oracle_matches_reference(case):
    z = golden()
    losses, gc, gb, gd = o.rpn(*rpn_inputs(z, case), g.rpn_cfg(RPN_CASES[case]))
    for pre, tol in (('', 1e-10), ('f32.', 1e-5)):
        assert rel(losses, z[f'{pre}{case}.tb']) <= tol
        for got, key in ((gc, 'g_cls_preds'), (gb, 'g_box_preds'), (gd, 'g_dir_cls_preds')):
            ref = z[f'{pre}{case}.{key}']
            assert rel(got.reshape(ref.shape), ref) <= tol, (pre, key)


@pytest.mark.parametrize('case', RCNN_CASES)
def test_rcnn_oracle_matches_reference(case):
    z = golden()
    branches, names = rcnn_branches(z, case)
    losses, grads = o.rcnn(branches, g.rcnn_cfg())
    for pre, tol in (('', 1e-10), ('f32.', 1e-5)) if case != 'T' else (('', 1e-10),):
        assert rel(losses[-1], z[f'{pre}{case}.tb'][0]) <= tol
        for b, (gc, gr) in zip(names, grads):
            for got, key in ((gc, 'g_cls'), (gr, 'g_reg')):
                ref = z[f'{pre}{case}.{key}.{b}']
                if not np.abs(ref).max():
                    assert not np.abs(got).max(), (pre, key, b)
                else:
                    assert rel(got, ref) <= tol, (pre, key, b)


def test_golden_covers_edge_cases():
    z = golden()
    y = z['L.box_cls_labels']
    assert {-1, 0, 1, 2} <= set(np.unique(y)) and not (y[1] > 0).any()      # ignored, folded, a scene without positives
    nan = np.isnan(z['L.box_reg_targets'])
    assert nan.any() and not nan[..., 6].any() and (nan.any(-1) & (y > 0)).any()
    assert (np.abs(z['L.cls_preds']) > 40).sum() >= 8
    assert (z['L.g_cls_preds'].reshape(y.shape)[y == -1] == 0).all()          # unweighted anchors: zero gradient
    assert set(np.unique(z['C3.box_cls_labels'])) == {-1, 0, 1, 2, 3}
    branches, names = rcnn_branches(z, 'R3')
    assert len(names) == 9 and names[:3] == ['targets_dict0', 'targets_dict_pi0', 'targets_dict_p0']
    fg = [int((t['reg_valid_mask'] > 0).sum()) for t, _ in branches]
    assert fg[6:] == [0, 0, 0] and min(fg[:6]) > 0                           # stage 2 without foreground
    assert not z['R3.g_reg.targets_dict2'].any()
    lab = z['R3.targets_dict0.rcnn_cls_labels']
    assert (lab == -1).any() and ((lab > 0) & (lab < 1)).any()                # ignored and soft labels
    x = z['R3.targets_dict0.rcnn_cls'][:, 0]
    sat = x > 40
    assert sat.any() and (z['R3.g_cls.targets_dict0'][sat] == 0).all()       # a saturated BCE has zero gradient
    t = {k: z[f'T.targets_dict0.{k}'] for k in g.RCNN_KEYS}
    assert (t['gt_of_rois_src'][0, 0, 3:5] == 0).all()                       # corner pairs tie
    assert t['rcnn_reg'][1, 0] == 0 and t['rcnn_reg'][1, 3] == 0 and t['gt_of_rois'][0, 1, 0] == 0
    assert t['gt_of_rois'][0, 1, 3] == t['rois'][0, 1, 3]                     # equal 1-D edges
    # every non-deliberate decision is at least MARGIN from its switch point
    for case, nc in RPN_CASES.items():
        ok = g.rpn_margins(z[f'{case}.cls_preds'], z[f'{case}.box_preds'], z[f'{case}.box_reg_targets'],
                           z[f'{case}.anchors_flat'], nc)
        assert ok[:, 8:].all() and ok[1].all()
    for case in ('R1', 'R3'):
        for t, _ in rcnn_branches(z, case)[0]:
            assert g.rcnn_margin_rows(t, g.rcnn_cfg())[6:].all()


def test_config_validation():
    from virconv_b200.head_losses import RCNNLossConfig, RPNLossConfig
    e = g.edict
    RPNLossConfig(e(g.RPN_CFG), 1)
    RCNNLossConfig(e(g.RCNN_CFG))
    for kw in (dict(OD_LOSS=True), dict(USE_MULTIHEAD=True),
               dict(LOSS_CONFIG=dict(g.RPN_CFG['LOSS_CONFIG'], REG_LOSS_TYPE='WeightedL1Loss')),
               dict(TARGET_ASSIGNER_CONFIG=dict(BOX_CODER='ResidualCoder',
                                                BOX_CODER_CONFIG={'encode_angle_by_sincos': True})),
               dict(LOSS_CONFIG=dict(LOSS_WEIGHTS=dict(g.RPN_CFG['LOSS_CONFIG']['LOSS_WEIGHTS'],
                                                       code_weights=[1.0] * 8)))):
        with pytest.raises(ValueError, match='AnchorHeadTemplate.get_loss'):
            RPNLossConfig(e(dict(g.RPN_CFG, **kw)), 1)
    lc = g.RCNN_CFG['LOSS_CONFIG']
    for kw in (dict(CLS_LOSS='CrossEntropy'), dict(REG_LOSS='l1')):
        with pytest.raises(ValueError, match='RoIHeadTemplate.get_loss'):
            RCNNLossConfig(e(dict(LOSS_CONFIG=dict(lc, **kw))))


@need_ref
@pytest.mark.parametrize('name', ['VirConv-L', 'VirConv-T', 'VirConv-S'])
def test_virconv_yamls_pass(name):
    from virconv_b200.head_losses import RCNNLossConfig, RPNLossConfig
    saved = dict(sys.modules)
    try:
        import virconv_b200.reference_env as renv
        from test_cpu_voxel_pool import REF
        renv.install(reference_root=REF)
        from pcdet.config import cfg, cfg_from_yaml_file
        cwd = os.getcwd()
        os.chdir(os.path.join(REF, 'tools'))
        try:
            cfg_from_yaml_file(os.path.join('cfgs', 'models', 'kitti', name + '.yaml'), cfg)
        finally:
            os.chdir(cwd)
        RPNLossConfig(cfg.MODEL.DENSE_HEAD, len(cfg.CLASS_NAMES))
        c = RCNNLossConfig(cfg.MODEL.ROI_HEAD)
        assert c.corner
    finally:
        _restore_modules(saved)


def test_ordered_anchors_match_reference_view():
    """the masked sets of AnchorHeadSingle.forward ([1, L, sizes, rotations, 7]): ordered_anchors (the assignment's
    order) is the loss's torch.cat(self.anchors, dim=-3).view(-1, 7); a full map is concatenated as the loss does"""
    from virconv_b200.anchor_targets import ordered_anchors
    from virconv_b200.head_losses import head_anchors
    gen = torch.Generator().manual_seed(0)
    for sets, shape in ((1, (1, 37, 1, 2, 7)), (3, (1, 21, 1, 2, 7)), (2, (1, 9, 2, 3, 7)), (1, (1, 5, 6, 1, 2, 7)),
                        (2, (1, 5, 6, 1, 2, 7))):
        anchors = [torch.randn(shape, generator=gen) for _ in range(sets)]
        ref = torch.cat(anchors, dim=-3).view(-1, 7)
        assert torch.equal(head_anchors(anchors), ref)
        if len(shape) == 5:
            assert torch.equal(ordered_anchors(anchors)[0], ref)


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


def test_branch_table_layout():
    """the ctypes mirror of vc_rcnn_branch: 9 pointers, 3 ints, a float"""
    import ctypes
    from virconv_b200.head_losses import _Branch
    assert ctypes.sizeof(_Branch) == 9 * 8 + 4 * 4 and _Branch.weight.offset == 9 * 8 + 12


@need_ref
def test_virconv_l_uses_fused_losses(monkeypatch):
    from virconv_b200 import head_losses
    saved = dict(sys.modules)
    try:
        model = _build_virconv_l(monkeypatch, use_fused_losses=True)
        assert type(model.dense_head).get_loss is head_losses.anchor_head_get_loss
        assert type(model.roi_head).get_loss is head_losses.roi_head_get_loss
        assert head_losses.RPNLossConfig(model.dense_head.model_cfg, model.dense_head.num_class).loc_weight == 2.0
        assert head_losses.RCNNLossConfig(model.roi_head.model_cfg).corner
    finally:
        _restore_modules(saved)
