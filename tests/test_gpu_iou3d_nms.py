"""GPU tests of the rotated-box IoU / NMS kernels (csrc/iou3d_nms.cu) against the outputs of the reference's own kernels
on seeded inputs (tests/golden/iou3d_ref_*.npz, recorded by oracle/iou3d_golden.py), the float64 restatement
oracle/iou3d.py, and restatements of the reference's per-scene Python loops."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import iou3d as o
from oracle import iou3d_golden as g

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')


def _golden(kind):
    return np.load(os.path.join(GOLDEN, f'iou3d_ref_{kind}.npz'))


def _defined(a, b, three_d=False):
    """pairs with a positive summed area (volume): where both boxes have none, the reference's IoU is the float rounding
    noise of a degenerate polygon divided by the 1e-8 (1e-6) floor — 7.8 for a zero-length box against itself —, not a
    value"""
    va, vb = a[:, 3] * a[:, 4] * (a[:, 5] if three_d else 1), b[:, 3] * b[:, 4] * (b[:, 5] if three_d else 1)
    return va[:, None] + vb[None] > 0


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize('case', ['rois512_gt48', 'cars300', 'edge'])
def test_pairwise_iou_vs_reference_fixtures_and_oracle(lib_built, case):
    from virconv_b200 import iou3d_nms
    ref = _golden('iou')
    a, b = g.iou_cases()[case]
    ov = iou3d_nms.boxes_overlap_bev(_d(a), _d(b)).cpu().numpy()
    iou = iou3d_nms.boxes_iou_bev(_d(a), _d(b)).cpu().numpy()
    iou3 = iou3d_nms.boxes_iou3d_gpu(_d(a), _d(b)).cpu().numpy()
    r_ov, r_iou, r_iou3 = ref[case + '_overlap'], ref[case + '_iou_bev'], ref[case + '_iou3d']
    d_ov = float((np.abs(ov - r_ov) / np.maximum(1.0, np.abs(r_ov))).max())
    d_iou = float(np.abs(iou - r_iou)[_defined(a, b)].max())
    d_iou3 = float(np.abs(iou3 - r_iou3)[_defined(a, b, True)].max())
    print(f'{case}: max |d overlap|/max(1,|ref|) {d_ov:.2e}, max |d iou_bev| {d_iou:.2e}, max |d iou3d| {d_iou3:.2e}')
    assert d_ov <= 2e-5 and d_iou <= 2e-5 and d_iou3 <= 2e-5
    assert np.abs(iou - o.matrix(a, b, o.iou_bev)).max() <= 2e-5
    assert np.abs(iou3 - o.matrix(a, b, o.iou3d)).max() <= 2e-5
    # the host entry point shares the geometry code: bit-identical
    assert np.array_equal(iou3d_nms.boxes_bev_iou_cpu(a, b), iou)


@pytest.mark.parametrize('n', g.NMS_SIZES)
def test_nms_keep_lists_identical_to_reference_fixtures(lib_built, n):
    from virconv_b200 import iou3d_nms
    from virconv_b200 import reference_env as renv
    ref = _golden('nms')
    boxes, sc = g.nms_boxes(n)
    for kind in ('rot', 'normal'):
        fn = iou3d_nms.nms_normal_gpu if kind == 'normal' else iou3d_nms.nms_gpu
        wrap = renv._nms_normal_gpu if kind == 'normal' else renv._nms_gpu
        for thresh in g.NMS_THRESHOLDS:
            idx, keep = ref[f'{kind}_{n}_{thresh}_idx'], ref[f'{kind}_{n}_{thresh}_keep']
            tb, ts = _d(boxes[idx]), _d(sc[idx])
            got, none = fn(tb, ts, thresh)
            assert none is None and got.dtype == torch.int64
            assert np.array_equal(got.cpu().numpy(), keep), (kind, thresh)
            # the iou3d_nms_cuda binding: boxes already sorted, CPU LongTensor `keep` written in place
            order = ts.sort(0, descending=True)[1]
            k = torch.LongTensor(len(idx))
            num = wrap(tb[order].contiguous(), k, thresh)
            assert np.array_equal(order[k[:num].cuda()].cpu().numpy(), keep), (kind, thresh)


def test_reference_env_binds_the_iou3d_nms_extension(lib_built):
    saved = dict(sys.modules)
    try:
        import virconv_b200.reference_env as renv
        renv.install()
        ext = sys.modules['pcdet.ops.iou3d_nms.iou3d_nms_cuda']
        a, b = g.iou_cases()['rois512_gt48']
        ta, tb = _d(a), _d(b)
        out = torch.zeros((len(a), len(b)), device='cuda')
        assert ext.boxes_iou_bev_gpu(ta, tb, out) == 1
        ref = _golden('iou')
        assert np.abs(out.cpu().numpy() - ref['rois512_gt48_iou_bev']).max() <= 2e-5
        assert ext.boxes_overlap_bev_gpu(ta, tb, out) == 1
        assert (np.abs(out.cpu().numpy() - ref['rois512_gt48_overlap']) <= 2e-5 * np.maximum(1.0, ref['rois512_gt48_overlap'])).all()
        cpu = torch.zeros((len(a), len(b)))
        assert ext.boxes_iou_bev_cpu(torch.from_numpy(a), torch.from_numpy(b), cpu) == 1
    finally:
        for k in list(sys.modules):
            if k not in saved and k.split('.')[0] in ('pcdet', 'spconv', 'cumm', 'easydict', 'tensorboardX',
                                                      'prefetch_generator', 'skimage'):
                del sys.modules[k]
        for k, v in saved.items():
            sys.modules[k] = v


def _ragged(seed, n_max=900, counts=(900, 0, 1)):
    boxes = np.zeros((len(counts), n_max, 9), np.float32)
    scores = np.zeros((len(counts), n_max), np.float32)
    for i, c in enumerate(counts):
        bx = g.cars(n_max, seed + i)
        boxes[i, :, :7] = bx
        boxes[i, :, 7:] = np.random.default_rng(seed + i).normal(size=(n_max, 2))
        scores[i] = g.scores(n_max, seed + 50 + i)
    return boxes, scores, np.array(counts, np.int32)


@pytest.mark.parametrize('normal', [False, True])
def test_nms_batched_equals_per_scene_nms(lib_built, normal):
    from virconv_b200 import iou3d_nms
    boxes, scores, counts = _ragged(5)
    tb, ts, tc = _d(boxes), _d(scores), _d(counts)
    fn = iou3d_nms.nms_normal_gpu if normal else iou3d_nms.nms_gpu
    for thresh, pre, post in ((0.8, 700, 512), (0.1, 900, 20), (0.75, 500, 50)):
        keep, num = iou3d_nms.nms_batched(tb, ts, tc, thresh, pre, post, normal=normal)
        if post == 20:
            assert int(num[0]) == 20          # truncated at post_maxsize
        keep, num = keep.cpu().numpy(), num.cpu().numpy()
        for b, c in enumerate(counts):
            if normal:
                o_ = ts[b, :c].sort(0, descending=True)[1][:pre]
                want = o_[fn(tb[b, :c, :7][o_].contiguous(), ts[b, :c][o_], thresh)[0]][:post]
            else:
                want = fn(tb[b, :c, :7].contiguous(), ts[b, :c], thresh, pre_maxsize=pre)[0][:post]
            want = want.cpu().numpy()
            assert num[b] == len(want), (b, thresh)
            assert np.array_equal(keep[b, :len(want)], want), (b, thresh)
            assert (keep[b, len(want):] == -1).all()
        assert num[1] == 0 and num[2] == 1


class _Cfg(dict):
    __getattr__ = dict.__getitem__


def _reference_proposal_layer(batch_box_preds, batch_cls_preds, cfg):
    """RoIHeadTemplate.proposal_layer (roi_head_template.py:84-116) + class_agnostic_nms (model_nms_utils.py:125-144)
    restated over the drop-in nms_gpu, one scene at a time"""
    from virconv_b200 import iou3d_nms
    B = batch_box_preds.shape[0]
    rois = batch_box_preds.new_zeros((B, cfg.NMS_POST_MAXSIZE, batch_box_preds.shape[-1]))
    roi_scores = batch_box_preds.new_zeros((B, cfg.NMS_POST_MAXSIZE))
    roi_labels = batch_box_preds.new_zeros((B, cfg.NMS_POST_MAXSIZE), dtype=torch.long)
    for index in range(B):
        box_preds, cls_preds = batch_box_preds[index], batch_cls_preds[index]
        cur_roi_scores, cur_roi_labels = torch.max(cls_preds, dim=1)
        box_scores_nms, indices = torch.topk(cur_roi_scores, k=min(cfg.NMS_PRE_MAXSIZE, cur_roi_scores.shape[0]))
        keep_idx, _ = getattr(iou3d_nms, cfg.NMS_TYPE)(box_preds[indices][:, 0:7], box_scores_nms, cfg.NMS_THRESH)
        selected = indices[keep_idx[:cfg.NMS_POST_MAXSIZE]]
        rois[index, :len(selected), :] = box_preds[selected]
        roi_scores[index, :len(selected)] = cur_roi_scores[selected]
        roi_labels[index, :len(selected)] = cur_roi_labels[selected]
    return rois, roi_scores, roi_labels + 1


def _proposal_inputs(seed, B=2, N=4200, C=7, ncls=3):
    boxes = np.stack([g.cars(N, seed + b) for b in range(B)])
    if C > 7:
        boxes = np.concatenate([boxes, np.random.default_rng(seed).normal(size=(B, N, C - 7)).astype(np.float32)], -1)
    rng = np.random.default_rng(seed + 100)
    cls = np.stack([rng.permutation(N * ncls).reshape(N, ncls) for _ in range(B)]).astype(np.float32) / (N * ncls)
    return _d(boxes), _d(cls)


CFGS = [_Cfg(MULTI_CLASSES_NMS=False, NMS_TYPE='nms_gpu', NMS_THRESH=0.8, NMS_PRE_MAXSIZE=4000, NMS_POST_MAXSIZE=512),
        _Cfg(MULTI_CLASSES_NMS=False, NMS_TYPE='nms_gpu', NMS_THRESH=0.75, NMS_PRE_MAXSIZE=2000, NMS_POST_MAXSIZE=50),
        _Cfg(MULTI_CLASSES_NMS=False, NMS_TYPE='nms_normal_gpu', NMS_THRESH=0.1, NMS_PRE_MAXSIZE=4096, NMS_POST_MAXSIZE=500)]


@pytest.mark.parametrize('ci', range(len(CFGS)))
def test_proposal_layer_equals_the_reference_loop(lib_built, ci):
    from virconv_b200 import iou3d_nms
    cfg = CFGS[ci]
    bp, cp = _proposal_inputs(30 + ci, C=9 if ci == 0 else 7)
    got = iou3d_nms.proposal_layer(bp, cp, cfg)
    want = _reference_proposal_layer(bp, cp, cfg)
    for x, y in zip(got, want):
        assert x.dtype == y.dtype and x.shape == y.shape
        assert torch.equal(x, y)
    assert int((got[2] > 1).sum()) > 0 or cfg.NMS_POST_MAXSIZE < 100


def test_proposal_layer_captured_in_a_cuda_graph(lib_built):
    """captured once, replayed on three seeded inputs copied into its static buffers: equal to the eager result (a
    successful capture is itself the check that nothing reads a device value on the host)"""
    from virconv_b200 import iou3d_nms
    cfg = CFGS[0]
    sb, sc = _proposal_inputs(40)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        iou3d_nms.proposal_layer(sb, sc, cfg)       # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = iou3d_nms.proposal_layer(sb, sc, cfg)
    for seed in (41, 42, 43):
        bp, cp = _proposal_inputs(seed)
        sb.copy_(bp)
        sc.copy_(cp)
        graph.replay()
        torch.cuda.synchronize()
        want = iou3d_nms.proposal_layer(bp, cp, cfg)
        for x, y in zip(out, want):
            assert torch.equal(x, y), seed


def test_empty_inputs(lib_built):
    from virconv_b200 import iou3d_nms
    z = torch.zeros((0, 7), device='cuda')
    b = _d(g.cars(5, 1))
    assert iou3d_nms.boxes_iou_bev(z, b).shape == (0, 5)
    assert iou3d_nms.boxes_iou3d_gpu(b, z).shape == (5, 0)
    keep, _ = iou3d_nms.nms_gpu(z, torch.zeros((0,), device='cuda'), 0.5)
    assert keep.numel() == 0
    keep, _ = iou3d_nms.nms_normal_gpu(z, torch.zeros((0,), device='cuda'), 0.5)
    assert keep.numel() == 0
    keep, num = iou3d_nms.nms_batched(torch.zeros((2, 0, 7), device='cuda'), torch.zeros((2, 0), device='cuda'),
                                      torch.zeros((2,), dtype=torch.int32, device='cuda'), 0.5, 100, 10)
    assert (keep == -1).all() and (num == 0).all()
    keep, num = iou3d_nms.nms_batched(b.view(1, 5, 7), torch.rand((1, 5), device='cuda'),
                                      torch.zeros((1,), dtype=torch.int32, device='cuda'), 0.5, 100, 10)
    assert (keep == -1).all() and (num == 0).all()
    rois, scores, labels = iou3d_nms.proposal_layer(torch.zeros((2, 0, 7), device='cuda'), torch.zeros((2, 0, 1), device='cuda'),
                                                    CFGS[1])
    assert rois.shape == (2, 50, 7) and (rois == 0).all() and (scores == 0).all() and (labels == 1).all()


def test_iou3d_nms_rejects_cpu_tensors(lib_built):
    from virconv_b200 import iou3d_nms
    b = torch.from_numpy(g.cars(4, 1))
    with pytest.raises(Exception):
        iou3d_nms.boxes_iou_bev(b, b)
    with pytest.raises(Exception):
        iou3d_nms.boxes_iou3d_gpu(b, b)
    with pytest.raises(Exception):
        iou3d_nms.nms_gpu(b, torch.rand(4), 0.5)
    with pytest.raises(Exception):
        iou3d_nms.proposal_layer(b.view(1, 4, 7), torch.rand(1, 4, 1), CFGS[1])
