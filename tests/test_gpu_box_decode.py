"""GPU tests of the box decoding and cascade stage transforms (rules R1-R3 of csrc/box_decode.cu): against the reference's
own float32 results (tests/golden/box_decode_ref.npz); at full size (2 x 70,400 anchors, 2 x 160 RoIs, three stages)
against oracle/box_decode.py and against the reference's control flow over torch on the same GPU; the box_preds
gradients against the closed form and torch.autograd of the float64 torch restatement; bit-identical repeats under
torch's deterministic flag; the drop-in methods under torch.cuda.set_sync_debug_mode('error'); a CUDA graph of an
eval-style stage loop."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import box_decode as o
from oracle import box_decode_golden as g
from test_cpu_box_decode import PERIOD, RCNN, RPN, golden, ulp_tol, within

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mb():
    sys.path.insert(0, os.path.join(ROOT, 'profiles'))
    import microbench_box_decode as mb
    return mb


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(t):
    return t.detach().cpu().numpy()


def ulps_of_magnitude(got, ref):
    """the largest error per column in ulp of that column's largest magnitude"""
    err = np.abs(got.astype(np.float64) - ref).reshape(-1, ref.shape[-1]).max(0)
    return (err / ulp_tol(ref, 1)).round(2).tolist()


@pytest.fixture()
def det_flag():
    saved = torch.are_deterministic_algorithms_enabled()
    yield
    torch.use_deterministic_algorithms(saved)


@pytest.mark.parametrize('case', RPN)
def test_rpn_matches_reference_golden(lib_built, case):
    from virconv_b200.box_decode import anchor_decode
    z = golden()
    box, anchors, dirs = z[f'{case}.box'], g.rpn_anchors(z, case), z[f'{case}.dir'] if f'{case}.dir' in z else None
    bp = _t(box).requires_grad_()
    out = anchor_decode(bp, _t(anchors), _t(dirs) if dirs is not None else None, g.DIR_OFFSET, g.DIR_LIMIT_OFFSET,
                        PERIOD)
    ref = z[f'f32.{case}.out']
    got = _np(out)
    assert within(got[..., :6], ref[..., :6], 2)
    amb = z[f'{case}.amb'] if dirs is not None else np.zeros(box.shape[:2], bool)
    assert np.array_equal(got[..., 6][~amb], ref[..., 6][~amb])      # the heading and so the direction label
    if f'{case}.g' in z:
        (d,) = torch.autograd.grad(out, [bp], _t(z[f'{case}.g']))
        assert within(_np(d), z[f'f32.{case}.dbox'], 2)


@pytest.mark.parametrize('case', RCNN)
def test_rcnn_matches_reference_golden(lib_built, case):
    from virconv_b200.box_decode import roi_decode
    z = golden()
    bp = _t(z[f'{case}.box']).requires_grad_()
    out = roi_decode(bp, _t(z[f'{case}.rois']))
    assert within(_np(out), z[f'f32.{case}.out'], 2)
    assert np.array_equal(_np(out)[..., 6], z[f'f32.{case}.out'][..., 6])
    (d,) = torch.autograd.grad(out, [bp], _t(z[f'{case}.g']))
    assert within(_np(d), z[f'f32.{case}.dbox'], 2)


@pytest.mark.parametrize('method', g.XT_METHODS)
def test_xtrans_matches_reference_golden(lib_built, method):
    from virconv_b200 import box_decode as bd
    z = golden()
    head = _mb()._HEAD
    boxes, tp = _t(z['X.boxes']), _t(z['X.tparam'])
    for R in (1, 2, 3):
        for i in range(3):
            key = f'f32.X.{method}.{R}.{g.clamp(i, R)}'
            got = _np(getattr(bd, method)(head, boxes, i, tp[:, :R].contiguous()))
            assert within(got, z[key], 2), key
            assert np.array_equal(got[..., 3:], z[key][..., 3:]), key           # sizes, flipped heading, extra columns


def test_full_size_matches_oracle_and_torch(lib_built):
    from virconv_b200 import box_decode as bd
    mb = _mb()
    dev = torch.device('cuda')
    gen = torch.Generator(device=dev).manual_seed(11)
    anchors = mb.kitti_anchors(dev)
    box = torch.randn(2, 70400, 7, device=dev, generator=gen) * 0.3
    dirs = torch.randn(2, 70400, 2, device=dev, generator=gen)
    dirs[:, :500, 1] = dirs[:, :500, 0]
    out = _np(bd.anchor_decode(box, anchors, dirs, 0.78539, 0.0, np.pi))
    bn, an, dn = _np(box), _np(anchors), _np(dirs)
    ref64 = o.anchor_decode(bn, an, dn, 0.78539, 0.0, np.pi)
    ref32 = o.anchor_decode(bn, an, dn, 0.78539, 0.0, np.pi, dtype=np.float32, div=False)
    assert within(out[..., :6], ref64[..., :6], 4)
    assert np.array_equal(out[..., 6], ref32[..., 6])
    with torch.no_grad():
        tref = _np(o.torch_anchor_decode(box, anchors, dirs))           # the reference's CUDA kernels
    assert np.array_equal(out[..., 6], tref[..., 6]) and within(out[..., :6], tref[..., :6], 2)
    rois = mb.kitti_rois(2, 160, 7, dev, ld=9)
    rbox = torch.randn(320, 7, device=dev, generator=gen) * 0.3
    rout = _np(bd.roi_decode(rbox, rois))
    assert within(rout, o.roi_decode(_np(rbox), _np(rois)), 4)
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            assert within(rout, _np(o.torch_roi_decode(rbox, rois)), 2)
            tp = mb.transform_param(dev)
            preds = mb.kitti_rois(2, 160, 8, dev)
            fused = mb.stage_loop('fused', rois, preds, tp)
            torch_ref = mb.stage_loop('reference', rois, preds, tp)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    assert len(fused) == 5                                           # pred at 0; score, pred at 1 and 2
    r = _np(rois)
    for i in range(3):                                               # the oracle's stage loop
        if i >= 1:
            r = o.xtrans(r, _np(tp), i - 1, i)
    for k, (a, b) in enumerate(zip(fused, torch_ref)):
        # stages 1 and 2 chain up to three rotations, each a few roundings apart from the reference's matmul
        assert within(_np(a), _np(b), 4), (k, ulps_of_magnitude(_np(a), _np(b)))
        assert np.array_equal(_np(a)[..., 3:], _np(b)[..., 3:]), k
    assert within(_np(fused[3]), o.xtrans(r, _np(tp), 2, 0), 4)           # roi_score_trans at stage 2


def test_backward_against_closed_form_and_autograd(lib_built):
    from virconv_b200 import box_decode as bd
    mb = _mb()
    dev = torch.device('cuda')
    gen = torch.Generator(device=dev).manual_seed(12)
    anchors = mb.kitti_anchors(dev)
    box = (torch.randn(2, 70400, 7, device=dev, generator=gen) * 0.3).requires_grad_()
    dirs = torch.randn(2, 70400, 2, device=dev, generator=gen)
    up = torch.randn(2, 70400, 7, device=dev, generator=gen)
    (d,) = torch.autograd.grad(bd.anchor_decode(box, anchors, dirs, 0.78539, 0.0, np.pi), [box], up)
    closed = o.anchor_decode_grad(_np(up), _np(box), _np(anchors))
    b64 = box.detach().double().requires_grad_()
    (auto,) = torch.autograd.grad(o.torch_anchor_decode(b64, anchors.double(), dirs.double()), [b64], up.double())
    assert within(_np(d), closed, 4) and within(_np(d), _np(auto), 4)
    rois = mb.kitti_rois(2, 160, 9, dev)
    rbox = (torch.randn(320, 7, device=dev, generator=gen) * 0.3).requires_grad_()
    rup = torch.randn(2, 160, 7, device=dev, generator=gen)
    (rd,) = torch.autograd.grad(bd.roi_decode(rbox, rois), [rbox], rup)
    r64 = rbox.detach().double().requires_grad_()
    (rauto,) = torch.autograd.grad(o.torch_roi_decode(r64, rois.double()), [r64], rup.double())
    assert within(_np(rd), o.roi_decode_grad(_np(rup), _np(rbox), _np(rois)), 4) and within(_np(rd), _np(rauto), 4)


def _all_outputs(mb, dev, seed):
    from virconv_b200 import box_decode as bd
    gen = torch.Generator(device=dev).manual_seed(seed)
    anchors = mb.kitti_anchors(dev)
    box = (torch.randn(2, 70400, 7, device=dev, generator=gen) * 0.3).requires_grad_()
    dirs = torch.randn(2, 70400, 2, device=dev, generator=gen)
    rois = mb.kitti_rois(2, 160, seed, dev)
    rbox = (torch.randn(320, 7, device=dev, generator=gen) * 0.3).requires_grad_()
    a = bd.anchor_decode(box, anchors, dirs, 0.78539, 0.0, np.pi)
    r = bd.roi_decode(rbox, rois)
    (da,) = torch.autograd.grad(a, [box], torch.ones_like(a))
    (dr,) = torch.autograd.grad(r, [rbox], torch.ones_like(r))
    with torch.no_grad():
        st = mb.stage_loop('fused', rois, r.detach(), mb.transform_param(dev))
    return [a.detach(), r.detach(), da, dr] + st


def test_bit_identical_repeats(lib_built, det_flag):
    mb = _mb()
    dev = torch.device('cuda')
    first = None
    for flag in (False, True, False, True):
        torch.use_deterministic_algorithms(flag)
        junk = torch.full((64 << 20,), float('nan'), device=dev)        # leaves dirty blocks in the cache
        del junk
        outs = _all_outputs(mb, dev, 31)
        if first is None:
            first = outs
        else:
            assert all(torch.equal(a, b) for a, b in zip(outs, first))


def test_drop_ins_never_synchronise(lib_built):
    from virconv_b200 import box_decode as bd
    mb = _mb()
    dev = torch.device('cuda')
    anchors = mb.kitti_anchors(dev)
    rpn = types.SimpleNamespace(anchors=[anchors.view(1, 35200, 1, 2, 7)], use_multihead=False,
                                box_coder=type('ResidualCoder', (), {'code_size': 7, 'encode_angle_by_sincos': False})(),
                                model_cfg=types.SimpleNamespace(DIR_OFFSET=0.78539, DIR_LIMIT_OFFSET=0.0, NUM_DIR_BINS=2))
    rcnn = types.SimpleNamespace(box_coder=rpn.box_coder, x_trans_train=mb._HEAD.x_trans_train)
    cls, box, dirs = (torch.randn(2, 35200, k, device=dev) for k in (2, 14, 4))
    rois = mb.kitti_rois(2, 160, 3, dev)
    tp = mb.transform_param(dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        bc, bb = bd.anchor_generate_predicted_boxes(rpn, 2, cls, box, dirs)
        rc, rb = bd.roi_generate_predicted_boxes(rcnn, 2, rois, torch.randn(320, 1, device=dev),
                                                 torch.randn(320, 7, device=dev))
        x = bd.roi_x_trans(rcnn, rois, 1, tp)
        s = bd.roi_score_trans(rcnn, x, 1, tp)
        p = bd.pred_x_trans(rcnn, rb, 2, tp)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert bc.shape == (2, 70400, 1) and bb.shape == (2, 70400, 7) and rc.shape == (2, 160, 1)
    assert x.shape == s.shape == p.shape == (2, 160, 7)
    with torch.no_grad():
        assert torch.equal(bb, bd.anchor_decode(box.view(2, -1, 7), anchors, dirs.view(2, -1, 2), 0.78539, 0.0,
                                                2 * np.pi / 2))
        assert torch.equal(p, bd.box_xtrans(rb, tp, 2, None))


def test_cuda_graph_stage_loop_replays_equal_eager(lib_built):
    from virconv_b200 import box_decode as bd
    mb = _mb()
    dev = torch.device('cuda')
    gen = torch.Generator(device=dev).manual_seed(41)
    head = types.SimpleNamespace(box_coder=type('ResidualCoder', (), {'code_size': 7, 'encode_angle_by_sincos': False})(),
                                 x_trans_train=mb._HEAD.x_trans_train)
    rois0 = mb.kitti_rois(2, 160, 5, dev)
    regs = [torch.randn(320, 7, device=dev, generator=gen) * 0.3 for _ in range(3)]
    tp = mb.transform_param(dev)

    def loop():       # the eval stage loop of multi_grid_pool_aggregation, its box arithmetic only
        rois, outs = rois0, []
        for i in range(3):
            if i >= 1:
                rois = bd.roi_x_trans(head, rois, i, tp)
                outs.append(bd.roi_score_trans(head, rois, i, tp))
            _, boxes = bd.roi_generate_predicted_boxes(head, 2, rois, torch.zeros(320, 1, device=dev), regs[i])
            outs.append(bd.pred_x_trans(head, boxes.clone(), i, tp))
            rois = boxes
        return outs

    with torch.no_grad():
        eager = [t.clone() for t in loop()]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                loop()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            outs = loop()
        for _ in range(3):
            for t in outs:
                t.fill_(float('nan'))
            graph.replay()
            torch.cuda.synchronize()
            assert all(torch.equal(a, b) for a, b in zip(outs, eager))


def test_argument_checks(lib_built):
    from virconv_b200.box_decode import anchor_decode, box_xtrans, roi_decode
    dev = torch.device('cuda')
    box, anc = torch.zeros(2, 10, 7, device=dev), torch.zeros(10, 7, device=dev)
    for args in ((box[..., :6], anc), (box, anc[:9]), (box.double(), anc)):
        with pytest.raises(ValueError, match='generate_predicted_boxes'):
            anchor_decode(*args)
    rois = torch.zeros(2, 10, 7, device=dev)
    for args in ((torch.zeros(19, 7, device=dev), rois), (torch.zeros(20, 7, device=dev), rois[..., :6])):
        with pytest.raises(ValueError, match='generate_predicted_boxes'):
            roi_decode(*args)
    tp = torch.zeros(2, 3, 3, device=dev)
    with pytest.raises(ValueError, match='roi_x_trans'):
        box_xtrans(rois, tp[:1], 0, 1)
    with pytest.raises(IndexError):
        box_xtrans(rois, tp, 3, None)
    wide = torch.randn(2, 10, 9, device=dev)
    assert torch.equal(box_xtrans(wide, tp + 1, 0, 1)[..., 7:], wide[..., 7:])
    assert torch.equal(box_xtrans(wide, tp + 1, -1, None), box_xtrans(wide, tp + 1, 2, None))
