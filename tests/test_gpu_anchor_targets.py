"""GPU tests of the RPN anchor mask and target assignment (csrc/anchor_targets.cu, virconv_b200/anchor_targets.py): the
kernels against the reference's own results (tests/golden/anchor_targets_ref.npz), VirConv-L's full map against the
float32 restatement oracle/anchor_targets.py, the GT capacity, the absence of host reads, and a CUDA-graph replay."""
import numpy as np
import pytest
import torch

from oracle import anchor_targets as o
from oracle import anchor_targets_golden as g
from test_cpu_anchor_targets import bits, case_inputs, golden

pytestmark = pytest.mark.gpu


def _assigner(case):
    from virconv_b200.anchor_targets import AxisAlignedTargetAssigner

    class Coder:
        code_size = 7
    sets = [g.CAR] if case == 'L' else g.SETS_T
    names = g.CLASS_NAMES_L if case == 'L' else g.CLASS_NAMES_T
    return AxisAlignedTargetAssigner(g.model_cfg(sets), names, Coder(), g.GRID, g.PCR)


def _anchor_sets(z, case, mask=None):
    """the generator's anchors per set, [1, Y, X, 1, 2, 7], masked like AnchorHeadSingle.forward"""
    sets = [g.CAR] if case == 'L' else g.SETS_T
    out = []
    for s, c in enumerate(sets):
        a = torch.from_numpy(o.anchors_from_shifts(z[f'{case}.x_shifts{s}'], z[f'{case}.y_shifts{s}'],
                                                   c['anchor_bottom_heights'], c['anchor_sizes'], c['anchor_rotations']))
        out.append(a.cuda() if mask is None else a.cuda()[:, mask])
    return out


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return float((np.abs(a.astype(np.float64) - b) / np.spacing(np.maximum(np.abs(b), np.float32(1e-30)))).max())


def test_mask_matches_reference(lib_built):
    from virconv_b200.anchor_targets import anchor_mask
    z = golden()
    m = anchor_mask(torch.from_numpy(z['L.points']).cuda(), g.PCR, g.GRID, g.FEATURE_SHAPE_L)
    assert m.dtype == torch.bool and m.is_cuda and tuple(m.shape) == (200, 176)
    assert np.array_equal(m.cpu().numpy(), z['L.mask'])


@pytest.mark.parametrize('case', ['L', 'T'])
def test_targets_match_reference(lib_built, case):
    z = golden()
    out = _assigner(case).assign_targets(_anchor_sets(z, case, torch.from_numpy(z[f'{case}.mask']).cuda()),
                                         torch.from_numpy(z[f'{case}.gt']).cuda())
    assert out['box_cls_labels'].dtype == torch.int32 and out['box_reg_targets'].shape[-1] == 7
    assert np.array_equal(out['box_cls_labels'].cpu().numpy(), z[f'{case}.box_cls_labels'])
    assert np.array_equal(bits(out['gt_ious'].cpu()), bits(z[f'{case}.gt_ious']))     # incl. -0.0
    assert np.array_equal(bits(out['reg_weights'].cpu()), bits(z[f'{case}.reg_weights']))
    t, ref = out['box_reg_targets'].cpu().numpy(), z[f'{case}.box_reg_targets']
    assert np.array_equal(t == 0, ref == 0) and _ulps(t, ref) <= 4


def _full_scene(seed, n_gt=40):
    """VirConv-L's whole 200 x 176 map (70,400 anchors), B = 2, n_gt car boxes per scene near anchors, some padding"""
    z = golden()
    anchors = _anchor_sets(z, 'L')
    rng = np.random.default_rng(seed)
    loc = anchors[0].reshape(-1, 7)[:, :2].cpu().numpy()
    gt = np.zeros((2, n_gt + 4, 8), np.float32)
    for b in range(2):
        for j in range(n_gt):
            gt[b, j] = g.box(rng, loc[rng.integers(len(loc))] + rng.normal(0, 0.6, 2).astype(np.float32), 1)
    gt[1, 7] = gt[1, 6]
    return anchors, gt


def _check_against_oracle(anchors, gt, out):
    a, sid = o.ordered([x.cpu().numpy() for x in anchors])
    labels, targets, reg, ious = o.assign(a, sid, gt, ['Car'], ['Car'], [0.6], [0.45])
    assert np.array_equal(out['box_cls_labels'].cpu().numpy(), labels)
    assert np.array_equal(bits(out['gt_ious'].cpu()), bits(ious))
    assert np.array_equal(bits(out['reg_weights'].cpu()), bits(reg))
    t = out['box_reg_targets'].cpu().numpy()
    assert np.array_equal(t == 0, targets == 0) and _ulps(t, targets) <= 4
    return labels


def test_full_size_against_oracle(lib_built):
    from virconv_b200 import scenes
    from virconv_b200.anchor_targets import anchor_mask
    anchors, gt = _full_scene(5)
    assigner = _assigner('L')
    out = assigner.assign_targets(anchors, torch.from_numpy(gt).cuda())
    assert out['box_cls_labels'].shape == (2, 70400)
    labels = _check_against_oracle(anchors, gt, out)
    assert (labels > 0).sum() > 200 and (labels < 0).sum() > 100
    # the masked subset, as AnchorHeadSingle.forward selects it from the points of two scenes
    pts = scenes.make_points_batch([0, 1], n_lidar=16384, n_virtual=80000, training=True).points
    mask = anchor_mask(torch.from_numpy(pts).cuda(), g.PCR, g.GRID, g.FEATURE_SHAPE_L)
    assert np.array_equal(mask.cpu().numpy(), o.anchor_mask(pts, *_mask_args()))
    masked = [x[:, mask] for x in anchors]
    _check_against_oracle(masked, gt, assigner.assign_targets(masked, torch.from_numpy(gt).cuda()))


def _mask_args():
    from virconv_b200.anchor_targets import mask_params
    return (*mask_params(g.PCR, g.GRID), 200, 176)


def test_gt_capacity_error(lib_built):
    from virconv_b200._lib import VirConvLibraryError
    from virconv_b200.anchor_targets import MAX_GT
    anchors, _ = _full_scene(1)
    gt = torch.zeros((1, MAX_GT + 1, 8), device='cuda')
    with pytest.raises(VirConvLibraryError, match=r'rc=-4'):
        _assigner('L').assign_targets(anchors, gt)
    out = _assigner('L').assign_targets(anchors, gt[:, :MAX_GT])         # at the limit: fine
    assert int((out['box_cls_labels'] != 0).sum()) == 0


def test_no_host_read(lib_built):
    from virconv_b200.anchor_targets import anchor_mask
    anchors, gt = _full_scene(2)
    pts = torch.from_numpy(golden()['L.points']).cuda()
    gt = torch.from_numpy(gt).cuda()
    assigner = _assigner('L')
    assigner.assign_targets(anchors, gt)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        anchor_mask(pts, g.PCR, g.GRID, g.FEATURE_SHAPE_L)
        assigner.assign_targets(anchors, gt)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    torch.cuda.synchronize()


def test_graph_replay_matches_eager(lib_built):
    from virconv_b200.anchor_targets import anchor_mask, assign_targets_batched, name_sets, ordered_anchors
    z = golden()
    anchors_sets = _anchor_sets(z, 'T')
    a, sid = ordered_anchors(anchors_sets)
    ns = name_sets(g.CLASS_NAMES_T, ['Car', 'Pedestrian', 'Cyclist'])
    thr = ([0.6, 0.5, 0.5], [0.45, 0.35, 0.35])
    B, N = 2, a.shape[0]
    gt_in = torch.zeros((B, g.M_GT, 8), device='cuda')
    pts_in = torch.zeros_like(torch.from_numpy(z['L.points'])).cuda()
    out = (torch.empty((B, N), dtype=torch.int32, device='cuda'), torch.empty((B, N, 7), device='cuda'),
           torch.empty((B, N), device='cuda'), torch.empty((B, N), device='cuda'))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                            # warm-up off the capturing stream
        assign_targets_batched(a, sid, gt_in, ns, *thr, out)
        anchor_mask(pts_in, g.PCR, g.GRID, g.FEATURE_SHAPE_L)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        assign_targets_batched(a, sid, gt_in, ns, *thr, out)
        mask_out = anchor_mask(pts_in, g.PCR, g.GRID, g.FEATURE_SHAPE_L)
    for seed in (3, 4):                                                   # new inputs in the same buffers
        rng = np.random.default_rng(seed)
        gt = np.zeros((B, g.M_GT, 8), np.float32)
        loc = a[:, :2].cpu().numpy()
        for b in range(B):
            for j in range(20 + 5 * b):
                gt[b, j] = g.box(rng, loc[rng.integers(len(loc))], int(rng.integers(1, 4)))
        gt_in.copy_(torch.from_numpy(gt))
        pts = z['L.points'].copy()
        pts[:, 1:3] += rng.normal(0, 3, (len(pts), 2)).astype(np.float32)
        pts_in.copy_(torch.from_numpy(pts))
        graph.replay()
        torch.cuda.synchronize()
        eager = _assigner('T').assign_targets(anchors_sets, gt_in)
        for k, got in zip(('box_cls_labels', 'box_reg_targets', 'reg_weights', 'gt_ious'), out):
            assert torch.equal(got.view(torch.int32), eager[k].view(torch.int32)), k
        assert torch.equal(mask_out, anchor_mask(pts_in, g.PCR, g.GRID, g.FEATURE_SHAPE_L))
        assert int((out[0] > 0).sum()) > 0
