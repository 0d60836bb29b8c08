"""GPU tests of the detection losses (csrc/head_losses.cu, virconv_b200/head_losses.py): the kernels against the
reference's own losses and autograd gradients (tests/golden/head_losses_ref.npz), full-size inputs against the float64
oracle, run-to-run bit equality, the absence of host reads, CUDA-graph replays of target assignment -> loss -> backward,
a non-unit incoming gradient, and the drop-in methods with their one host read."""
import types
import warnings

import numpy as np
import pytest
import torch

from oracle import head_losses as o
from oracle import head_losses_golden as g
from test_cpu_head_losses import RCNN_CASES, RPN_CASES, golden, rcnn_branches, rel, rpn_inputs

pytestmark = pytest.mark.gpu


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run_rpn(inputs, cfg, grad_out=None):
    from virconv_b200.head_losses import rpn_loss
    cls, box, dirp, labels, tgt, anchors = inputs
    preds = [cu(cls).requires_grad_(), cu(box).requires_grad_(), None if dirp is None else cu(dirp).requires_grad_()]
    loss, stats = rpn_loss(preds[0], preds[1], preds[2], cu(labels), cu(tgt), cu(anchors), cfg)
    live = [p for p in preds if p is not None]
    grads = torch.autograd.grad(loss, live, grad_out)
    return stats.cpu().numpy(), [gr.cpu().numpy() for gr in grads]


def torch_branches(branches):
    out = []
    for t, w in branches:
        d = {k: cu(v) for k, v in t.items()}
        d['rcnn_cls'].requires_grad_()
        d['rcnn_reg'].requires_grad_()
        out.append((d, w))
    return out


def run_rcnn(branches, cfg, grad_out=None):
    from virconv_b200.head_losses import rcnn_loss
    tb = torch_branches(branches)
    loss, stats = rcnn_loss(tb, cfg)
    preds = [x for t, _ in tb for x in (t['rcnn_cls'], t['rcnn_reg'])]
    grads = torch.autograd.grad(loss, preds, grad_out)
    return stats.cpu().numpy(), [gr.cpu().numpy() for gr in grads]


@pytest.mark.parametrize('case', list(RPN_CASES))
def test_rpn_matches_reference(lib_built, case):
    z = golden()
    stats, (gc, gb, gd) = run_rpn(rpn_inputs(z, case), g.rpn_cfg(RPN_CASES[case]))
    assert np.abs(stats - z[f'{case}.tb']).max() <= 1e-5 * np.abs(z[f'{case}.tb']).max()
    for got, key in ((gc, 'g_cls_preds'), (gb, 'g_box_preds'), (gd, 'g_dir_cls_preds')):
        ref = z[f'{case}.{key}']
        assert got.shape == ref.shape and rel(got, ref) <= 1e-5, key
        assert (got[ref == 0] == 0).all(), key
    B, N = z[f'{case}.box_cls_labels'].shape
    y = z[f'{case}.box_cls_labels']
    assert (gc.reshape(B, N, -1)[y == -1] == 0).all()                             # unweighted anchors
    assert (gb.reshape(B, N, 7)[y <= 0] == 0).all() and (gd.reshape(B, N, -1)[y <= 0] == 0).all()
    nan = np.isnan(z[f'{case}.box_reg_targets'])
    assert (gb.reshape(B, N, 7)[nan] == 0).all()                                  # NaN targets


@pytest.mark.parametrize('case', RCNN_CASES)
def test_rcnn_matches_reference(lib_built, case):
    z = golden()
    branches, names = rcnn_branches(z, case)
    stats, grads = run_rcnn(branches, g.rcnn_cfg())
    assert abs(stats[-1] - z[f'{case}.tb'][0]) <= 1e-5 * abs(z[f'{case}.tb'][0])
    ref_losses, _ = o.rcnn(branches, g.rcnn_cfg())
    assert rel(stats, ref_losses) <= 1e-5
    for k, b in enumerate(names):
        for got, key in ((grads[2 * k], 'g_cls'), (grads[2 * k + 1], 'g_reg')):
            ref = z[f'{case}.{key}.{b}']
            assert got.shape == ref.shape
            assert np.abs(got - ref).max() <= 1e-5 * max(np.abs(ref).max(), 1e-30), (key, b)
            assert (got[ref == 0] == 0).all(), (key, b)
        t = branches[k][0]
        sat = np.abs(t['rcnn_cls'][:, 0]) > 40
        sat &= (1 / (1 + np.exp(-t['rcnn_cls'][:, 0].astype(np.float64)))) == 1.0
        assert (grads[2 * k][sat] == 0).all()                                       # saturated BCE
        assert (grads[2 * k + 1][t['reg_valid_mask'].reshape(-1) <= 0] == 0).all()


def full_rpn(seed, B=2, L=35200, A=2, nc=1):
    rng = np.random.default_rng(seed)
    N = L * A
    anchors = np.zeros((N, 7), np.float32)
    anchors[:, :2] = rng.uniform(-40, 70, (N, 2))
    anchors[:, 3:6] = (3.9, 1.6, 1.56)
    anchors[:, 6] = np.tile([0.0, 1.57], L)
    labels = rng.choice([-1, 0, 0, 0, 0, 0, 0, 0, 0, 1], (B, N)).astype(np.int32)
    tgt = np.where((labels > 0)[..., None], rng.normal(0, 0.3, (B, N, 7)), 0).astype(np.float32)
    return (rng.normal(0, 2, (B, L, A * nc)).astype(np.float32), rng.normal(0, 0.3, (B, L, A * 7)).astype(np.float32),
            rng.normal(0, 1.5, (B, L, A * 2)).astype(np.float32), labels, tgt, anchors)


def test_rpn_full_size_against_oracle(lib_built):
    inputs = full_rpn(1)                                                            # 2 x 70,400 anchors
    cfg = g.rpn_cfg(1)
    stats, grads = run_rpn(inputs, cfg)
    ref = o.rpn(*inputs, cfg)
    assert rel(stats, ref[0]) <= 1e-5
    for got, r in zip(grads, ref[1:]):
        assert rel(got, r.reshape(got.shape)) <= 1e-5


def virconv_t_branches(seed, B=2, R=160):
    rng = np.random.default_rng(seed)
    cfg = g.rcnn_cfg()
    out = []
    for i in range(3):
        t = g.target_set(rng, B, R, 0.4)
        for w in (1.0, 0.5, 0.5):
            n = B * R
            d = dict(t, rcnn_cls=rng.normal(0, 2, (n, 1)).astype(np.float32),
                     rcnn_reg=rng.normal(0, 0.15, (n, 7)).astype(np.float32))
            out.append((d, w))
    return out, cfg


def test_rcnn_virconv_t_against_oracle(lib_built):
    branches, cfg = virconv_t_branches(2)                                          # 9 branches of 2 x 160
    stats, grads = run_rcnn(branches, cfg)
    ref, rgrads = o.rcnn(branches, cfg)
    assert rel(stats, ref) <= 1e-5
    for k, (gc, gr) in enumerate(rgrads):
        assert rel(grads[2 * k], gc) <= 1e-5 and rel(grads[2 * k + 1], gr) <= 1e-5


def test_bit_identical_runs(lib_built):
    inputs = full_rpn(3)
    cfg = g.rpn_cfg(1)
    a, b = run_rpn(inputs, cfg), run_rpn(inputs, cfg)
    assert a[0].tobytes() == b[0].tobytes() and all(x.tobytes() == y.tobytes() for x, y in zip(a[1], b[1]))
    branches, rcfg = virconv_t_branches(4)
    a, b = run_rcnn(branches, rcfg), run_rcnn(branches, rcfg)
    assert a[0].tobytes() == b[0].tobytes() and all(x.tobytes() == y.tobytes() for x, y in zip(a[1], b[1]))


def test_non_unit_grad_output(lib_built):
    z = golden()
    go = torch.tensor(-2.5, device='cuda')
    _, grads = run_rpn(rpn_inputs(z, 'L'), g.rpn_cfg(1), go)
    for got, key in zip(grads, ('g_cls_preds', 'g_box_preds', 'g_dir_cls_preds')):
        assert rel(got, -2.5 * z[f'L.{key}']) <= 1e-5
    branches, names = rcnn_branches(z, 'R1')
    _, grads = run_rcnn(branches, g.rcnn_cfg(), go)
    for k, b in enumerate(names):
        assert rel(grads[2 * k + 1], -2.5 * z[f'R1.g_reg.{b}']) <= 1e-5


def test_no_host_read(lib_built):
    from virconv_b200.head_losses import rcnn_loss, rpn_loss
    z = golden()
    cls, box, dirp, labels, tgt, anchors = (cu(a) for a in rpn_inputs(z, 'L'))
    preds = [t.requires_grad_() for t in (cls, box, dirp)]
    tb = torch_branches(rcnn_branches(z, 'R3')[0])
    rcfg, pcfg = g.rcnn_cfg(), g.rpn_cfg(1)
    rpn_loss(*preds, labels, tgt, anchors, pcfg)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        l1, _ = rpn_loss(*preds, labels, tgt, anchors, pcfg)
        l2, _ = rcnn_loss(tb, rcfg)
        (l1 + l2).backward()
    finally:
        torch.cuda.set_sync_debug_mode('default')
    torch.cuda.synchronize()
    assert preds[0].grad is not None and tb[0][0]['rcnn_reg'].grad is not None


def _graph_equals_eager(step, fill, outs):
    fill(1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    captured = list(outs())                                                         # the graph's own output tensors
    for seed in (2, 3):
        fill(seed)
        graph.replay()
        torch.cuda.synchronize()
        got = [t.clone() for t in captured]
        step()
        torch.cuda.synchronize()
        for a, b in zip(got, outs()):
            assert torch.equal(a, b)


def test_graph_rpn_targets_loss_backward(lib_built):
    from virconv_b200.anchor_targets import assign_targets_batched
    from virconv_b200.head_losses import rpn_loss
    cfg = g.rpn_cfg(1)
    B, L, M = 2, 4000, 16
    N = 2 * L
    anchors = torch.zeros((N, 7), device='cuda')
    sid = torch.zeros(N, dtype=torch.int32, device='cuda')
    gt = torch.zeros((B, M, 8), device='cuda')
    cls = torch.zeros((B, L, 2), device='cuda', requires_grad=True)
    box = torch.zeros((B, L, 14), device='cuda', requires_grad=True)
    dirp = torch.zeros((B, L, 4), device='cuda', requires_grad=True)
    out = (torch.empty((B, N), dtype=torch.int32, device='cuda'), torch.empty((B, N, 7), device='cuda'),
           torch.empty((B, N), device='cuda'), torch.empty((B, N), device='cuda'))
    res = {}

    def step():
        for p in (cls, box, dirp):
            p.grad = None
        assign_targets_batched(anchors, sid, gt, [1], [0.6], [0.45], out)
        loss, stats = rpn_loss(cls, box, dirp, out[0], out[1], anchors, cfg)
        loss.backward()
        res['stats'] = stats
        res['g'] = (cls.grad, box.grad, dirp.grad)

    def fill(seed):
        rng = np.random.default_rng(seed)
        a = np.zeros((N, 7), np.float32)
        a[:, 0], a[:, 1] = rng.uniform(0, 70, N), rng.uniform(-40, 40, N)
        a[:, 2], a[:, 3:6], a[:, 6] = -1.78, (3.9, 1.6, 1.56), np.tile([0.0, 1.57], L)
        anchors.copy_(torch.from_numpy(a))
        gg = np.zeros((B, M, 8), np.float32)
        for b in range(B):
            idx = rng.integers(0, N, 12)
            gg[b, :12, :7] = a[idx] + rng.normal(0, 0.2, (12, 7)).astype(np.float32)
            gg[b, :12, 7] = 1
        gt.copy_(torch.from_numpy(gg))
        with torch.no_grad():
            for p in (cls, box, dirp):
                p.copy_(torch.from_numpy(rng.normal(0, 1, p.shape).astype(np.float32)))

    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        _graph_equals_eager(step, fill, lambda: (res['stats'],) + res['g'] + out)
    assert int((out[0] > 0).sum()) > 0 and float(res['g'][1].abs().max()) > 0


def test_graph_roi_targets_loss_backward(lib_built):
    from oracle import roi_targets_golden as rg
    from virconv_b200.head_losses import rcnn_loss
    from virconv_b200.reference_env import EasyDict
    from virconv_b200.roi_targets import SamplerConfig, empty_outputs, roi_targets_batched
    scfg = SamplerConfig(EasyDict(rg.CASES['L']))
    cfg = g.rcnn_cfg()
    B, M, G = 2, 512, 40
    rois_in = torch.zeros((B, M, 7), device='cuda')
    scores = torch.zeros((B, M), device='cuda')
    labels = torch.ones((B, M), dtype=torch.int64, device='cuda')
    gt = torch.zeros((B, G, 8), device='cuda')
    u = (torch.zeros((B, M), device='cuda'), torch.zeros((B, scfg.R), device='cuda'), torch.zeros(1, device='cuda'))
    out = empty_outputs(B, scfg.R, 7, 8, 'cuda')
    n = B * scfg.R
    preds = [torch.zeros((n, 1), device='cuda', requires_grad=True), torch.zeros((n, 7), device='cuda', requires_grad=True)]
    res = {}

    def step():
        for p in preds:
            p.grad = None
        roi_targets_batched(scfg, rois_in, scores, labels, gt, u, out)
        t = dict(out, rcnn_cls=preds[0], rcnn_reg=preds[1])
        loss, stats = rcnn_loss([(t, 1.0), (t, 0.5)], cfg)
        loss.backward()
        res['stats'] = stats
        res['g'] = (preds[0].grad, preds[1].grad)

    def fill(seed):
        rng = np.random.default_rng(seed)
        gg = np.zeros((B, G, 8), np.float32)
        rr = np.zeros((B, M, 7), np.float32)
        for b in range(B):
            rows = [rg.gt_box(rng, 1) for _ in range(30)]
            gg[b, :30] = np.stack(rows)
            for i in range(M):
                rr[b, i] = rg.near(rng, rows[rng.integers(30)], rng.choice([0.1, 0.4, 1.0]))
        gt.copy_(torch.from_numpy(gg))
        rois_in.copy_(torch.from_numpy(rr))
        scores.copy_(torch.from_numpy(rng.random((B, M), dtype=np.float32)))
        for x in u:
            x.copy_(torch.from_numpy(rng.random(tuple(x.shape), dtype=np.float32)))
        with torch.no_grad():
            preds[0].copy_(torch.from_numpy(rng.normal(0, 2, (n, 1)).astype(np.float32)))
            preds[1].copy_(torch.from_numpy(rng.normal(0, 0.15, (n, 7)).astype(np.float32)))

    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        _graph_equals_eager(step, fill, lambda: (res['stats'],) + res['g'] + tuple(out.values()))
    assert int((out['reg_valid_mask'] > 0).sum()) > 0 and float(res['g'][1].abs().max()) > 0


def _count_syncs(fn):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('warn')
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter('always')
            r = fn()
    finally:
        torch.cuda.set_sync_debug_mode('default')
    return r, sum('synchroniz' in str(x.message) for x in w)


def test_drop_in_methods(lib_built):
    from virconv_b200.head_losses import anchor_head_get_loss, roi_head_get_loss
    z = golden()
    cls, box, dirp, labels, tgt, flat = rpn_inputs(z, 'L')
    anchors = [cu(a) for a in z['L.anchors']]                                      # [1, L, 1, 2, 7] per set
    rpn = types.SimpleNamespace(model_cfg=g.edict(g.RPN_CFG), num_class=1, anchors=anchors,
                                forward_ret_dict={'cls_preds': cu(cls).requires_grad_(), 'box_preds': cu(box),
                                                  'dir_cls_preds': cu(dirp), 'box_cls_labels': cu(labels),
                                                  'box_reg_targets': cu(tgt)})
    anchor_head_get_loss(rpn)
    (loss, tb), n = _count_syncs(lambda: anchor_head_get_loss(rpn))
    assert n == 1 and list(tb) == ['rpn_loss_cls', 'rpn_loss_loc', 'rpn_loss_dir', 'rpn_loss']
    ref = o.rpn(cls, box, dirp, labels, tgt, flat, g.rpn_cfg(1))[0]
    assert rel(list(tb.values()), ref) <= 1e-5 and all(type(v) is float for v in tb.values())
    assert torch.equal(rpn.forward_ret_dict['box_cls_labels'].cpu(), torch.from_numpy(labels))   # labels not written
    branches, names = rcnn_branches(z, 'R3')
    frd = {b: t for b, (t, _) in zip(names, torch_branches(branches))}
    roi = types.SimpleNamespace(model_cfg=g.edict(g.RCNN_CFG), forward_ret_dict=frd)
    roi_head_get_loss(roi)
    (loss, tb2), n = _count_syncs(lambda: roi_head_get_loss(roi, {'x': 1.0}))
    assert n == 1 and list(tb2) == ['x', 'rcnn_loss']
    assert abs(tb2['rcnn_loss'] - z['R3.tb'][0]) <= 1e-5 * abs(z['R3.tb'][0])
