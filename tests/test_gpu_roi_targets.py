"""GPU tests of the RoI target sampling (csrc/roi_targets.cu, virconv_b200/roi_targets.py): the kernels against the
reference's own results (tests/golden/roi_targets_ref.npz), full-size scenes against the float32 restatement
oracle/roi_targets.py fed with vc_boxes_iou3d's own IoU matrix, the capacity error, the status word, the absence of host
reads, a CUDA-graph replay of the proposal NMS followed by the sampling, and the law of the drop-in layer's draws."""
import numpy as np
import pytest
import torch

from oracle import roi_targets as o
from oracle import roi_targets_golden as g
from test_cpu_roi_targets import EXACT, case_inputs, close_canonical, golden

pytestmark = pytest.mark.gpu


def _cfg(case_or_dict):
    from virconv_b200.reference_env import EasyDict
    from virconv_b200.roi_targets import SamplerConfig
    return SamplerConfig(EasyDict(g.CASES[case_or_dict] if isinstance(case_or_dict, str) else case_or_dict))


def _run(cfg, rois, scores, labels, gt, u_fg, u_bg, u_hs):
    from virconv_b200.roi_targets import empty_outputs, roi_targets_batched
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()    # noqa: E731
    B = rois.shape[0]
    out = empty_outputs(B, cfg.R, rois.shape[-1], gt.shape[-1], 'cuda')
    roi_targets_batched(cfg, c(rois), c(scores), c(labels), c(gt), (c(u_fg), c(u_bg), c(u_hs)), out)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _iou_gpu(a, b):
    """vc_boxes_iou3d's own matrix"""
    from virconv_b200 import iou3d_nms
    return iou3d_nms.boxes_iou3d_gpu(torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda(),
                                     torch.from_numpy(np.ascontiguousarray(b, np.float32)).cuda()).cpu().numpy()


@pytest.mark.parametrize('case', ['L', 'S', 'C'])
def test_matches_reference(lib_built, case):
    z = golden()
    out = _run(_cfg(case), *case_inputs(z, case))
    for k in EXACT:
        assert out[k].dtype == z[f'{case}.{k}'].dtype and np.array_equal(out[k], z[f'{case}.{k}']), k
    assert np.abs(out['gt_iou_of_rois'] - z[f'{case}.gt_iou_of_rois']).max() <= 2e-5
    assert np.abs(out['rcnn_cls_labels'] - z[f'{case}.rcnn_cls_labels']).max() <= 4e-5
    assert close_canonical(out['gt_of_rois'], z[f'{case}.gt_of_rois'], z[f'{case}.rois'], z[f'{case}.gt_of_rois_src'])
    assert out['status'][0] == 0


def _scene(seed, B=2, M=512, n_gt=40, G=44, classes=(1,)):
    """B scenes of n_gt boxes (+ zero padding) and M proposals: near the GTs, far away, and zero-padded with label 1"""
    rng = np.random.default_rng(seed)
    gt = np.zeros((B, G, 8), np.float32)
    rois = np.zeros((B, M, 7), np.float32)
    labels = np.ones((B, M), np.int64)
    for b in range(B):
        rows = [g.gt_box(rng, int(rng.choice(classes))) for _ in range(n_gt)]
        gt[b, :n_gt] = np.stack(rows)
        for i in range(M - M // 16):
            r = rows[rng.integers(n_gt)]
            rois[b, i] = g.near(rng, r, rng.choice([0.1, 0.4, 1.0, 3.0])) if i % 8 else g.far(rng)
            labels[b, i] = int(r[7])
    scores = rng.random((B, M)).astype(np.float32)
    return rois, scores, labels, gt


def _uniforms(seed, B, M, R, n_cls):
    rng = np.random.default_rng(seed + 1000)
    return (rng.random((B, max(M, R)), dtype=np.float32), rng.random((B, R), dtype=np.float32),
            rng.random(n_cls, dtype=np.float32))


def _check_against_oracle(cfg_case, rois, scores, labels, gt, seed=0):
    cfg = _cfg(cfg_case)
    u = _uniforms(seed, rois.shape[0], rois.shape[1], cfg.R, cfg.n_cls)
    out = _run(cfg, rois, scores, labels, gt, *u)
    ref = o.sample(g.cfg_of(cfg_case) if isinstance(cfg_case, str) else cfg_case, rois, scores, labels, gt, *u, _iou_gpu)
    for k in EXACT + ('gt_iou_of_rois', 'rcnn_cls_labels'):
        assert out[k].dtype == ref[k].dtype and np.array_equal(out[k].view(np.uint8), ref[k].view(np.uint8)), k
    assert close_canonical(out['gt_of_rois'], ref['gt_of_rois'], ref['rois'], ref['gt_of_rois_src'])
    assert out['status'][0] == ref['status']
    return out, ref


@pytest.mark.parametrize('M', [512, 160])
def test_full_size_against_oracle(lib_built, M):
    out, ref = _check_against_oracle('L', *_scene(5 + M, M=M))
    assert (out['reg_valid_mask'] > 0).sum() > 40 and (ref['sampled'] >= 0).all()
    _check_against_oracle('C', *_scene(7 + M, M=M, classes=(1, 2, 3)), seed=1)


def test_foreground_only_scene_against_oracle(lib_built):
    rois, scores, labels, gt = _scene(3, B=2, M=160, n_gt=10, G=10)
    rng = np.random.default_rng(3)
    for i in range(160):                                                 # scene 1: every RoI a near copy of a GT
        r = gt[1, rng.integers(10)]
        rois[1, i] = r[:7] + np.float32(0.01) * rng.normal(size=7).astype(np.float32)
        labels[1, i] = 1
    out, ref = _check_against_oracle('L', rois, scores, labels, gt)
    assert (out['gt_iou_of_rois'][1] >= 0.55).all() and len(np.unique(ref['sampled'][1])) < 160   # with replacement


def test_capacity_error(lib_built):
    from virconv_b200._lib import VirConvLibraryError
    from virconv_b200.roi_targets import MAX_GT, MAX_ROIS
    cfg = _cfg('L')
    for M, G in ((MAX_ROIS + 1, 8), (16, MAX_GT + 1)):
        rois, scores, labels, gt = _scene(1, B=1, M=M, n_gt=4, G=G)
        with pytest.raises(VirConvLibraryError, match=r'rc=-4'):
            _run(cfg, rois, scores, labels, gt, *_uniforms(1, 1, M, cfg.R, 1))
    rois, scores, labels, gt = _scene(1, B=1, M=MAX_ROIS, n_gt=40, G=MAX_GT)          # at the limits: fine
    out = _run(cfg, rois, scores, labels, gt, *_uniforms(1, 1, MAX_ROIS, cfg.R, 1))
    assert out['status'][0] == 0 and (out['reg_valid_mask'] > 0).any()


def test_status_for_a_scene_without_candidates(lib_built):
    from virconv_b200.roi_targets import check_status
    rois, scores, labels, gt = _scene(2, B=2, M=64, n_gt=6, G=8)
    gt[1, :6, 7] = 3                                       # scene 1: class 3 has no threshold entry -> never fg / hard
    rng = np.random.default_rng(2)
    for i in range(64):
        rois[1, i] = gt[1, rng.integers(6), :7]             # IoU 1 with a class-3 GT: not easy either
        labels[1, i] = 3
    out, ref = _check_against_oracle('L', rois, scores, labels, gt)
    assert out['status'][0] == 1 and ref['status'] == 1
    for k in ('rois', 'gt_of_rois', 'gt_of_rois_src', 'gt_iou_of_rois', 'reg_valid_mask', 'roi_labels'):
        assert not out[k][1].any(), k
    assert out['rois'][0].any()
    with pytest.raises(NotImplementedError, match='FG=0, BG=0'):
        check_status(torch.from_numpy(out['status']).cuda())
    check_status(torch.zeros(1, dtype=torch.int32, device='cuda'))


def _batch(rois, scores, labels, gt):
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()    # noqa: E731
    return {'batch_size': rois.shape[0], 'rois': c(rois), 'roi_scores': c(scores), 'roi_labels': c(labels),
            'gt_boxes': c(gt), 'gt_boxes1': c(gt[:, ::-1].copy())}


def test_no_host_read(lib_built):
    from virconv_b200.roi_targets import ProposalTargetLayer, assign_targets
    import types
    batch = _batch(*_scene(4))
    layer = ProposalTargetLayer(g.cfg_of('L'))
    head = types.SimpleNamespace(proposal_target_layers=[layer, layer])
    layer(batch)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        fwd = layer(batch)
        tgt = assign_targets(head, batch, 1, enable_dif=True)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    torch.cuda.synchronize()
    assert set(fwd) == {'rois', 'gt_of_rois', 'gt_iou_of_rois', 'roi_scores', 'roi_labels', 'reg_valid_mask',
                        'rcnn_cls_labels'}
    assert list(tgt) == list(fwd) + ['gt_of_rois_src']
    assert tgt['roi_labels'].dtype == torch.int64 and tgt['reg_valid_mask'].dtype == torch.int64
    assert tgt['gt_of_rois'].shape == (2, 160, 8) and tgt['rcnn_cls_labels'].dtype == torch.float32
    assert (tgt['gt_of_rois'][..., 6].abs() <= np.float32(np.pi / 2)).all()


def test_graph_replay_matches_eager(lib_built):
    from virconv_b200 import iou3d_nms
    from virconv_b200.roi_targets import empty_outputs, roi_targets_batched
    cfg = _cfg('L')
    nms_cfg = {'MULTI_CLASSES_NMS': False, 'NMS_TYPE': 'nms_gpu', 'NMS_THRESH': 0.8, 'NMS_PRE_MAXSIZE': 2048,
               'NMS_POST_MAXSIZE': 512}
    B, N, G = 2, 3000, 44
    box_in = torch.zeros((B, N, 7), device='cuda')
    cls_in = torch.zeros((B, N, 1), device='cuda')
    gt_in = torch.zeros((B, G, 8), device='cuda')
    u_in = (torch.zeros((B, 512), device='cuda'), torch.zeros((B, cfg.R), device='cuda'), torch.zeros(1, device='cuda'))
    out = empty_outputs(B, cfg.R, 7, 8, 'cuda')

    def step():
        rois, scores, labels = iou3d_nms.proposal_layer(box_in, cls_in, nms_cfg)
        roi_targets_batched(cfg, rois, scores, labels, gt_in, u_in, out)
        return rois, scores, labels

    def fill(seed):
        rois, _, _, gt = _scene(seed, M=N, G=G)
        rng = np.random.default_rng(seed)
        box_in.copy_(torch.from_numpy(rois))
        cls_in.copy_(torch.from_numpy(rng.normal(size=(B, N, 1)).astype(np.float32)))
        gt_in.copy_(torch.from_numpy(gt))
        for u, n in zip(u_in, _uniforms(seed, B, 512, cfg.R, 1)):
            u.copy_(torch.from_numpy(n))
    fill(1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                            # warm-up off the capturing stream
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    for seed in (3, 4):                                                   # new inputs in the same buffers
        fill(seed)
        graph.replay()
        torch.cuda.synchronize()
        got = {k: v.clone() for k, v in out.items()}
        step()
        torch.cuda.synchronize()
        for k in got:
            assert torch.equal(got[k], out[k]), k
        assert int((got['reg_valid_mask'] > 0).sum()) > 0


def test_drawing_law(lib_built):
    """the drop-in layer over a few hundred draws: no foreground RoI twice in a scene, each candidate picked with
    frequency min(F, nf) / nf within 5 sigma"""
    from virconv_b200.roi_targets import ProposalTargetLayer
    rois, scores, labels, gt = _scene(9, M=512)
    layer = ProposalTargetLayer(g.cfg_of('L'))
    batch = _batch(rois, scores, labels, gt)
    cfg = layer._cfg
    trials = 300
    for b in range(2):
        g_b = gt[b, :o.trimmed_count(gt[b])]
        ov, asg = o.match(rois[b], labels[b], g_b, _iou_gpu)
        fg = np.nonzero((ov >= np.float32(0.55)) & (g_b[asg, -1] == 1))[0]
        assert len(fg) > cfg.F, len(fg)
    counts = np.zeros((2, 512))
    torch.manual_seed(0)
    for _ in range(trials):
        out = layer(batch)
        # foreground rows come first; the RoI index is recovered from its (unique) score
        s = out['roi_scores'][:, :cfg.F].cpu().numpy()
        for b in range(2):
            idx = np.nonzero(scores[b][None, :] == s[b][:, None])[1]
            assert len(idx) == cfg.F and len(np.unique(idx)) == cfg.F
            counts[b, idx] += 1
    for b in range(2):
        g_b = gt[b, :o.trimmed_count(gt[b])]
        ov, asg = o.match(rois[b], labels[b], g_b, _iou_gpu)
        fg = np.nonzero((ov >= np.float32(0.55)) & (g_b[asg, -1] == 1))[0]
        p = cfg.F / len(fg)
        sigma = np.sqrt(trials * p * (1 - p))
        assert counts[b, np.setdiff1d(np.arange(512), fg)].sum() == 0
        assert np.abs(counts[b, fg] - trials * p).max() < 5 * sigma
