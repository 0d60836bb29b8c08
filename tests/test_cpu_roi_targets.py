"""RoI target sampling without a GPU: the float32 restatement oracle/roi_targets.py against the reference's own
`ProposalTargetLayer.forward` + `RoIHeadTemplate.assign_targets` (tests/golden/roi_targets_ref.npz, recorded by
oracle/roi_targets_golden.py), the reference-RNG shims against the law they state, the constructor's limits, the
library's new symbols, and — where the reference's sources exist — the VirConv-L detector built with
`reference_env.install(use_fused_roi_targets=True)`."""
import os
import sys

import numpy as np
import pytest

from oracle import roi_targets as o
from oracle import roi_targets_golden as g
from test_cpu_voxel_pool import _build_virconv_l, _restore_modules, need_ref

SYMS = ('vc_roi_targets_ws_bytes', 'vc_roi_targets')
EXACT = ('rois', 'roi_scores', 'roi_labels', 'gt_of_rois_src', 'reg_valid_mask')


def golden():
    return np.load(os.path.join(os.path.dirname(__file__), 'golden', 'roi_targets_ref.npz'))


def case_inputs(z, case):
    """(rois, roi_scores, roi_labels, gt, u_fg, u_bg, u_hs) of a golden case"""
    return tuple(z[f'{case}.{k}'] for k in ('rois_in', 'roi_scores_in', 'roi_labels_in', 'gt', 'u_fg', 'u_bg', 'u_hs'))


def close_canonical(got, ref, rois, src, ulps=4, atol=1e-6):
    """gt_of_rois: within `ulps` of the reference, or `atol` absolute near 0 (the reference rotates with a matmul).  x'
    and y' are x cos - y sin and x sin + y cos of the centre offsets, which can cancel: their ulp is taken at the larger
    of the result and |x| + |y|."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float32)
    scale = np.abs(ref)
    d = (np.abs(src[..., 0] - rois[..., 0]) + np.abs(src[..., 1] - rois[..., 1])).astype(np.float32)
    scale[..., 0:2] = np.maximum(scale[..., 0:2], d[..., None])
    err = np.abs(got - ref)
    return bool(np.all((err <= ulps * np.spacing(scale).astype(np.float64)) | (err <= atol)))


@pytest.mark.parametrize('case', ['L', 'S', 'C'])
def test_oracle_matches_reference(case):
    z = golden()
    out = o.sample(g.cfg_of(case), *case_inputs(z, case), g.iou_f32)
    for k in EXACT:
        assert out[k].dtype == z[f'{case}.{k}'].dtype and np.array_equal(out[k], z[f'{case}.{k}']), k
    assert np.abs(out['gt_iou_of_rois'] - z[f'{case}.gt_iou_of_rois']).max() <= 2e-5
    assert np.abs(out['rcnn_cls_labels'] - z[f'{case}.rcnn_cls_labels']).max() <= 4e-5
    assert close_canonical(out['gt_of_rois'], z[f'{case}.gt_of_rois'], z[f'{case}.rois'], z[f'{case}.gt_of_rois_src'])
    assert out['status'] == 0


def test_golden_covers_edge_cases():
    z = golden()
    rois, scores, labels, gt, *_ = case_inputs(z, 'L')
    n0 = o.trimmed_count(gt[0])
    assert n0 < gt.shape[1] and (gt[0, :n0].sum(1) == 0).any()                # ragged, with an interior zero row
    u, c = np.unique(gt[0, :n0], axis=0, return_counts=True)
    assert (c[u[:, 3] > 0] > 1).any()                                         # a duplicated GT
    assert (rois[:, -32:] == 0).all() and (labels[:, -32:] == 1).all()        # zero-padded proposals, label 1
    assert (labels == 2).any() and not (gt[..., 7] == 2).any()                # a RoI class without GT
    dup = np.nonzero((gt[0, :n0, None] == gt[0, None, :n0]).all(-1).sum(1) > 1)[0]
    assert np.isin(z['L.gt_of_rois_src'][0], gt[0, dup[0]]).all(1).any()      # a tie was assigned (to its first row)
    assert z['L.reg_valid_mask'].sum() > 0 and (z['L.gt_iou_of_rois'] < 0.1).any()
    # case S: fg + easy only, no fg, all-zero GT (one zero row), only hard
    iou = z['S.gt_iou_of_rois']
    assert (iou[0] >= 0.5).sum() == 80 and (iou[0] < 0.1).sum() == 80
    assert (iou[1] < 0.5).all() and ((iou[1] >= 0.1).any() and (iou[1] < 0.1).any())
    assert not z['S.gt'][2].any() and (iou[2] == 0).all()
    assert ((iou[3] >= 0.1) & (iou[3] < 0.5)).all()
    # case C: two threshold classes, class 3 never sampled above CLS_BG_THRESH_LO
    src = z['C.gt_of_rois_src']
    assert {1, 2} <= set(np.unique(src[..., 7]).astype(int))
    assert (z['C.gt'][..., 7] == 3).any() and (z['C.gt_iou_of_rois'][src[..., 7] == 3] < 0.1).all()


def test_rng_shims_state_the_law():
    rng = np.random.default_rng(0)
    n, k, trials = 9, 4, 6000
    counts = np.zeros((k, n))
    for _ in range(trials):
        d = g.Draws(rng.random((1, 16), dtype=np.float32), rng.random((1, 8), dtype=np.float32),
                    rng.random(2, dtype=np.float32))
        d.new_scene()
        perm = d.permutation(n)
        assert sorted(perm) == list(range(n))                                 # a permutation
        counts[np.arange(k), perm[:k]] += 1
        assert np.all(np.diff(d.u_fg[0, perm]) >= 0)                          # ascending keys
        for high, size in ((3, 5), (7, 3)):
            r = d.torch_randint(low=0, high=high, size=(size,)).numpy()
            assert r.dtype == np.int64 and len(r) == size and r.min() >= 0 and r.max() < high
        assert d.pos == 8
        assert 0 <= d.np_randint(0, 2) < 2 and 0 <= d.np_randint(0, 4) < 4
        f = np.floor(d.rand(16) * n)
        assert f.min() >= 0 and f.max() < n and np.array_equal(f.astype(np.int64), o.draw(d.u_fg[0], n))
    # each position of the prefix is uniform over the n items: a sample without replacement
    p = 1.0 / n
    sigma = np.sqrt(trials * p * (1 - p))
    assert np.abs(counts - trials * p).max() < 5 * sigma


def test_draw_edges():
    assert o.draw(np.float32(0.0), 5) == 0
    assert o.draw(np.nextafter(np.float32(1), np.float32(0)), 5) == 4
    assert o.draw(np.float32(0.2), 5) == 1                                    # 0.2f * 5 in float64 is above 1


def test_trimming_rules():
    gt = np.zeros((5, 8), np.float32)
    assert o.trimmed_count(gt) == 1
    gt[3, 7] = 1                                                              # only a class: kept (class column counts)
    assert o.trimmed_count(gt) == 4
    gt[3, 7] = 0
    gt[2, 0] = 1
    assert o.trimmed_count(gt) == 3


def test_canonical_heading_fold():
    rois = np.zeros((4, 7), np.float32)
    rois[:, 6] = [0.0, -0.5, 4.0, 0.0]
    gt = np.zeros((4, 8), np.float32)
    gt[:, 0] = 1.0
    gt[:, 6] = [3.0, -0.5, 4.0, -2.0]
    out = o.canonical(rois, gt)
    h = out[:, 6]
    assert np.all(np.abs(h) <= np.float32(np.pi / 2))
    assert abs(h[0] - (3.0 - np.pi)) < 1e-6 and h[1] == 0 and h[2] == 0
    assert abs(out[1, 0] - np.cos(-(2 * np.pi - 0.5))) < 1e-6                  # rotated by -remainder(ry, 2 pi)


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
    from virconv_b200.roi_targets import MAX_CLASSES, ProposalTargetLayer
    ProposalTargetLayer(g.cfg_of('L'))
    ProposalTargetLayer(g.cfg_of('C'))
    bad = [dict(CLS_SCORE_TYPE='roi_iou'), dict(CLS_SCORE_TYPE='cls'), dict(SAMPLE_ROI_BY_EACH_CLASS=False),
           dict(REG_FG_THRESH=[0.55] * (MAX_CLASSES + 1), CLS_FG_THRESH=[0.75] * (MAX_CLASSES + 1),
                CLS_BG_THRESH=[0.25] * (MAX_CLASSES + 1), HARD_SAMPLING_THRESH=[0.5] * (MAX_CLASSES + 1),
                HARD_SAMPLING_RATIO=[0.5] * (MAX_CLASSES + 1))]
    from virconv_b200.reference_env import EasyDict
    for kw in bad:
        with pytest.raises(ValueError, match='reference class'):
            ProposalTargetLayer(EasyDict(dict(g.CFG_L, **kw)))


@need_ref
def test_virconv_l_head_uses_fused_layer(monkeypatch):
    from virconv_b200 import roi_targets
    saved = dict(sys.modules)
    try:
        keys_default = list(_build_virconv_l(monkeypatch).state_dict())
    finally:
        _restore_modules(saved)
    try:
        model = _build_virconv_l(monkeypatch, use_fused_roi_targets=True)
        head = model.roi_head
        assert type(head).__name__ == 'TEDMHead'
        assert len(head.proposal_target_layers) == 6
        assert all(type(p) is roi_targets.ProposalTargetLayer for p in head.proposal_target_layers)
        assert type(head).assign_targets is roi_targets.assign_targets
        assert roi_targets._reference_assign_targets is not None
        assert head.proposal_target_layers[0]._cfg.R == 160 and head.proposal_target_layers[0]._cfg.hard_sampling
        assert list(model.state_dict()) == keys_default
    finally:
        _restore_modules(saved)
