"""Deterministic mode (torch.use_deterministic_algorithms): the kernels through their C ABI — bit-identical across calls,
grid sizes and CTA caps, and close to the atomic kernels — and whole training steps of the plan executor, bit-identical
from run to run."""
import copy
import ctypes
import warnings

import numpy as np
import pytest
import torch

from oracle import gather2d as og
from oracle import rulebook as orb
from oracle.testing import fill_module, rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG8 = dict(CFG, LAYER_DISCARD_RATE=0.15, MM=True)


def _lib():
    from virconv_b200 import _lib as L
    return L, L.load()


def _st():
    from virconv_b200 import ops
    return ops._stream()


def _err():
    from virconv_b200 import ops
    return ops.tc_error_flag(DEV)


def _bf(t):
    return t.to(torch.bfloat16).float()


def _coords(rng, n, batch, shape, unique=True):
    c = np.stack([rng.integers(0, batch, n)] + [rng.integers(0, s, n) for s in shape], 1).astype(np.int32)
    if unique:
        c = np.unique(c, axis=0)
        rng.shuffle(c)
    return np.ascontiguousarray(c)


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=DEV)


@pytest.fixture
def det_mode():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize('cin,cout', [(16, 16), (32, 64), (64, 64), (8, 16)])
def test_wgrad_tc_det(lib_built, cin, cout):
    from virconv_b200 import ops
    L, lib = _lib()
    rng = np.random.default_rng(cin + cout)
    shape = [30, 120, 120]
    c = _coords(rng, 60000, 2, shape)
    n = c.shape[0]
    rb = ops.build_subm_rulebook(torch.from_numpy(c).to(DEV), 2, shape, 3)
    torch.manual_seed(cin)
    x, dy = _bf(torch.randn(n, cin, device=DEV)), _bf(torch.randn(n, cout, device=DEV))
    xb, dyb = x.to(torch.bfloat16), dy.to(torch.bfloat16)
    ref = torch.empty(cout, 27, cin, device=DEV)
    ws = _ws(lib.vc_conv_wgrad_ws_bytes(n, cin, cout, 27))
    L.check(lib.vc_conv_wgrad_f32(x.data_ptr(), dy.data_ptr(), rb.nbr.data_ptr(), ref.data_ptr(), n, cin, cout, 27, ws.data_ptr(),
                                  ws.numel(), _st()), 'vc_conv_wgrad_f32')
    wsd = _ws(lib.vc_conv_wgrad_tc_det_ws_bytes(n, cin, cout, 27))
    outs = []
    try:
        for cap in (0, 7, 33, 132, 0):
            L.check(lib.vc_conv_wgrad_tc3_config(1, cap), 'vc_conv_wgrad_tc3_config')
            dw = torch.empty(cout, 27, cin, device=DEV)
            L.check(lib.vc_conv_wgrad_tc_det(xb.data_ptr(), dyb.data_ptr(), rb.nbr.data_ptr(), dw.data_ptr(), n, cin, cout, 27,
                                             wsd.data_ptr(), wsd.numel(), _err().data_ptr(), _st()), 'vc_conv_wgrad_tc_det')
            outs.append(dw)
    finally:
        lib.vc_conv_wgrad_tc3_config(1, 0)
    # float64 reference of the same bf16-rounded operands
    nbr = rb.nbr.long()
    want = torch.zeros(27, cin, cout, dtype=torch.float64, device=DEV)
    for k in range(27):
        o = torch.nonzero(nbr[k] >= 0).squeeze(1)
        want[k] = x.double()[nbr[k, o]].t() @ dy.double()[o]
    want = want.permute(2, 0, 1)
    torch.cuda.synchronize()
    assert int(_err().item()) == 0
    # (fp32 accumulation over ~60 k rows: both kernels sit 1-2.5e-6 from the float64 sum, measured on an H100)
    assert rel_err(outs[0].double().cpu(), want.cpu()) < 3e-6
    assert rel_err(ref.double().cpu(), want.cpu()) < 3e-6
    assert rel_err(outs[0].cpu(), ref.cpu()) < 3e-6
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def _rb2d(co, shape):
    from virconv_b200 import ops
    L, lib = _lib()
    n = co.shape[0]
    ci = torch.from_numpy(co).to(DEV)
    nbr = torch.empty(9, n, dtype=torch.int32, device=DEV)
    pn = torch.empty(9, dtype=torch.int32, device=DEV)
    rep = torch.empty(n, dtype=torch.int32, device=DEV)
    ws = _ws(lib.vc_subm_rulebook_ws_bytes(n))
    L.check(lib.vc_subm_rulebook_rep(ci.data_ptr(), n, 2, 2, L.host_i32(shape), L.host_i32([3, 3]), L.host_i32([1, 1]),
                                     nbr.data_ptr(), pn.data_ptr(), rep.data_ptr(), ws.data_ptr(), ws.numel(), _st()),
            'vc_subm_rulebook_rep')
    return nbr, rep


def _gather2d(tc, dout, w, nbr, rep, n, n_dev, cin, cout):
    L, lib = _lib()
    din = torch.full((n, cin), 7.0, device=DEV)
    ws = _ws(lib.vc_conv_dgrad_gather2d_ws_bytes(n, cin, cout, 9))
    nd = n_dev.data_ptr() if n_dev is not None else None
    if tc:
        rc = lib.vc_conv_dgrad_gather2d_tc(dout.to(torch.bfloat16).data_ptr(), w.data_ptr(), nbr.data_ptr(), rep.data_ptr(),
                                           din.data_ptr(), n, nd, cin, cout, 9, ws.data_ptr(), ws.numel(), _err().data_ptr(), _st())
    else:
        rc = lib.vc_conv_dgrad_gather2d_f32(dout.data_ptr(), w.data_ptr(), nbr.data_ptr(), rep.data_ptr(), din.data_ptr(), n, nd,
                                            cin, cout, 9, ws.data_ptr(), ws.numel(), _st())
    L.check(rc, 'vc_conv_dgrad_gather2d')
    return din


@pytest.mark.parametrize('c', [8, 16, 32, 64])
def test_gather2d_dgrad(lib_built, c):
    L, lib = _lib()
    rng = np.random.default_rng(c)
    shape = [48, 36]
    co = _coords(rng, 20000, 2, shape, unique=False)
    n = co.shape[0]
    nbr, rep = _rb2d(co, shape)
    assert np.array_equal(nbr.cpu().numpy(), orb.subm_rulebook(co, shape, 3))
    assert np.array_equal(rep.cpu().numpy(), og.representatives(co, shape))
    torch.manual_seed(c)
    w = torch.randn(c, 3, 3, c, device=DEV) * 0.1
    dout = torch.randn(n, c, device=DEV)
    # fp32: against the scatter dgrad
    sc = torch.zeros(n, c, device=DEV)
    ws = _ws(lib.vc_conv_ws_bytes(c, c, 9))
    L.check(lib.vc_conv_dgrad_scatter_f32(dout.data_ptr(), w.data_ptr(), nbr.data_ptr(), sc.data_ptr(), n, c, c, 9, ws.data_ptr(),
                                          ws.numel(), _st()), 'vc_conv_dgrad_scatter_f32')
    g32 = _gather2d(False, dout, w, nbr, rep, n, None, c, c)
    assert rel_err(g32.cpu(), sc.cpu()) < 1e-5
    assert torch.equal(g32, _gather2d(False, dout, w, nbr, rep, n, None, c, c))
    # bf16: against the float64 oracle fed the kernel's own rounded operands (dout, S and the weights in bf16)
    gtc = _gather2d(True, dout, w, nbr, rep, n, None, c, c)
    torch.cuda.synchronize()
    assert int(_err().item()) == 0
    db = _bf(dout).cpu().numpy()
    rep_np = rep.cpu().numpy().astype(np.int64)
    s = np.zeros((n, c), np.float32)
    np.add.at(s, rep_np, db)
    s = _bf(torch.from_numpy(s)).numpy()
    want = og.gather_dgrad(db, _bf(w).reshape(c, 9, c).cpu().numpy(), nbr.cpu().numpy(), rep_np, s)
    assert rel_err(gtc.cpu(), torch.from_numpy(want).float()) < 1e-4
    assert torch.equal(gtc, _gather2d(True, dout, w, nbr, rep, n, None, c, c))
    # static-mode tails: capacity rows with a device count; the valid rows are the bits of the exact call, the tail is zero
    cap = n + 300
    nbr_c = torch.full((9, cap), -1, dtype=torch.int32, device=DEV)
    nbr_c[:, :n] = nbr
    rep_c = torch.full((cap,), -1, dtype=torch.int32, device=DEV)
    rep_c[:n] = rep
    dout_c = torch.randn(cap, c, device=DEV)
    dout_c[:n] = dout
    n_dev = torch.tensor([n], dtype=torch.int32, device=DEV)
    for tc, exact in ((False, g32), (True, gtc)):
        got = _gather2d(tc, dout_c, w, nbr_c, rep_c, cap, n_dev, c, c)
        assert torch.equal(got[:n], exact)
        assert not got[n:].any()


@pytest.mark.parametrize('precision', [0, 1])
def test_bn_sums_det(lib_built, precision):
    from virconv_b200 import ops
    L, lib = _lib()
    rng = np.random.default_rng(5)
    shape = [30, 120, 120]
    c = _coords(rng, 60000, 2, shape)
    n = c.shape[0]
    rb = ops.build_subm_rulebook(torch.from_numpy(c).to(DEV), 2, shape, 3)
    torch.manual_seed(5)
    x = torch.randn(n, 32, device=DEV)
    xin = x.to(torch.bfloat16) if precision else x
    w = torch.randn(64, 3, 3, 3, 32, device=DEV) * 0.1
    out = torch.empty(n, 64, device=DEV)
    ws = _ws(lib.vc_conv_fwd_det_ws_bytes(n, 32, 64, 27))
    sums = []
    try:
        for ctas in ((0, 1, 2, 0) if precision else (0, 0)):
            L.check(lib.vc_conv_tc2_config(ctas), 'vc_conv_tc2_config')
            s = torch.empty(2, 64, dtype=torch.float64, device=DEV)
            L.check(lib.vc_conv_fwd_det(precision, xin.data_ptr(), w.data_ptr(), rb.nbr.data_ptr(), out.data_ptr(), n, 32, 64, 27,
                                        s.data_ptr(), ws.data_ptr(), ws.numel(), _err().data_ptr(), _st()), 'vc_conv_fwd_det')
            sums.append(s)
    finally:
        lib.vc_conv_tc2_config(0)
    torch.cuda.synchronize()
    o = out.double()
    want = torch.stack([o.sum(0), (o * o).sum(0)])
    assert float((sums[0] - want).abs().max() / want.abs().max()) < 1e-6
    for s in sums[1:]:
        assert torch.equal(s, sums[0])


def test_bn_bwd_det(lib_built):
    L, lib = _lib()
    torch.manual_seed(9)
    n, c = 70001, 32
    x, dy = torch.randn(n, c, device=DEV), torch.randn(n, c, device=DEV)
    stats = torch.cat([torch.rand(c) + 0.5, torch.randn(c) * 0.1, torch.randn(c) * 0.1, torch.rand(c) + 0.5]).to(DEV)
    gamma = torch.rand(c, device=DEV) + 0.5
    ws = _ws(lib.vc_bn_bwd_det_ws_bytes(n, c))
    res = []
    try:
        for fused in (1, 1, 0):
            L.check(lib.vc_set_bn_fused(fused), 'vc_set_bn_fused')
            dx, dg, db = torch.empty(n, c, device=DEV), torch.empty(c, device=DEV), torch.empty(c, device=DEV)
            L.check(lib.vc_bn_relu_bwd_det_f32(dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), stats.data_ptr(), dx.data_ptr(), None,
                                               dg.data_ptr(), db.data_ptr(), n, c, 1, ws.data_ptr(), ws.numel(), _st()),
                    'vc_bn_relu_bwd_det_f32')
            res.append((dx, dg, db))
    finally:
        lib.vc_set_bn_fused(1)
    bs = torch.zeros(2, c, dtype=torch.float64, device=DEV)
    dx0, dg0, db0 = torch.empty(n, c, device=DEV), torch.empty(c, device=DEV), torch.empty(c, device=DEV)
    L.check(lib.vc_bn_relu_bwd_f32(dy.data_ptr(), x.data_ptr(), None, gamma.data_ptr(), stats.data_ptr(), dx0.data_ptr(), None,
                                   dg0.data_ptr(), db0.data_ptr(), n, c, 1, bs.data_ptr(), _st()), 'vc_bn_relu_bwd_f32')
    torch.cuda.synchronize()
    for r in res[1:]:
        for a, b in zip(r, res[0]):
            assert torch.equal(a, b)
    assert rel_err(res[0][0].cpu(), dx0.cpu()) < 1e-5
    assert rel_err(res[0][1].cpu(), dg0.cpu()) < 1e-5 and rel_err(res[0][2].cpu(), db0.cpu()) < 1e-5


# ------------------------------------------------------------------------------------------------ whole steps
def _batch(ids, n_lidar=4096, n_virtual=9000, max_voxels=7000):
    from virconv_b200 import scenes
    b = scenes.make_batch(ids, n_lidar=n_lidar, n_virtual=n_virtual, max_voxels=max_voxels, training=True)
    return {'voxel_features': torch.from_numpy(b.voxel_features.copy()).to(DEV),
            'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).to(DEV), 'batch_size': b.batch_size, 'calib': b.calib,
            'aug_param': torch.from_numpy(b.aug_param.copy())}


def _loss(named):
    from virconv_b200.graph import masked_mean
    return sum(masked_mean(t) for t in named.values())


def _record(model, out_named, loss):
    rec = {'loss': loss.detach().clone()}
    for k, t in out_named.items():
        rec['f:' + k] = t.features.detach().clone()
        rec['i:' + k] = t.indices.clone()
    for k, v in model.named_parameters():
        rec['g:' + k] = v.grad.clone()
    for k, v in model.named_buffers():
        rec['b:' + k] = v.clone()
    return rec


def _dirty():
    """park blocks full of non-zero bytes in the caching allocator, like a training loop's other work does"""
    hold = [torch.full((32 << 20,), float(torch.randint(1, 100, ()).item()), device=DEV) for _ in range(32)]
    del hold


def _step_l(model, state, batch):
    model.load_state_dict(state)
    for p in model.parameters():
        p.grad = None
    out = model(dict(batch))
    named = dict(out['multi_scale_3d_features'])
    named['out'] = out['encoded_spconv_tensor']
    loss = _loss(named)
    loss.backward()
    torch.cuda.synchronize()
    return _record(model, named, loss)


@pytest.mark.parametrize('precision,training', [('bf16', True), ('fp32', True), ('bf16', False)])
def test_virconv_l_step_bit_identical(lib_built, precision, training, monkeypatch):
    """two steps on the same batch, also after other work left the caching allocator's blocks dirty"""
    from virconv_b200 import executor
    from virconv_b200.backbone import VirConvL8x
    runs = []
    note = executor.note_last_run
    monkeypatch.setattr(executor, 'note_last_run', lambda model, run: (runs.append(run), note(model, run)))
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], precision=precision)
    fill_module(m, 666)
    m.to(DEV).train(training)
    state = copy.deepcopy(m.state_dict())
    batch = _batch([3, 4])
    torch.use_deterministic_algorithms(True)
    try:
        _dirty()
        a = _step_l(m, state, batch)
        _dirty()
        det, det_bytes = runs[-1].deterministic_bytes()
        b = _step_l(m, state, batch)
    finally:
        torch.use_deterministic_algorithms(False)
    assert det and det_bytes > 0
    assert int(_err().item()) == 0
    bad = {k: float((a[k].double() - b[k].double()).abs().max()) for k in a if not torch.equal(a[k], b[k])}
    assert not bad, bad
    off = _step_l(m, state, batch)          # flag off: the atomic kernels, within the existing tolerances
    gtol = 3e-2 if precision == 'bf16' else 2e-4
    for k in a:
        if k.startswith('i:') or k.endswith('num_batches_tracked'):
            assert torch.equal(a[k], off[k]), k
        elif k.startswith('g:'):
            assert rel_err(a[k].cpu(), off[k].cpu()) < gtol, k
        else:
            assert rel_err(a[k].cpu().float(), off[k].cpu().float()) < 1e-4, k


def test_graphed_step_replays_bit_identical(lib_built, det_mode):
    from virconv_b200.backbone import VirConvL8x
    from virconv_b200.graph import GraphedStep
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], precision='bf16')
    fill_module(m, 666)
    m.to(DEV).train()
    batch = _batch([5, 6])

    def loss_fn(out):
        named = dict(out['multi_scale_3d_features'])
        named['out'] = out['encoded_spconv_tensor']
        return _loss(named)

    step = GraphedStep(m, loss_fn)
    params = dict(m.named_parameters())
    got = []
    for _ in range(6):
        loss = step(batch)
        torch.cuda.synchronize()
        got.append((loss.detach().clone(), {k: v.grad.clone() for k, v in params.items()}))
    assert int(_err().item()) == 0
    for loss, g in got[2:]:
        assert torch.equal(loss, got[1][0])
        for k in g:
            assert torch.equal(g[k], got[1][1][k]), k


def test_virconv8x_paper_stvd_bit_identical(lib_built, det_mode):
    from virconv_b200 import scenes
    from virconv_b200.backbone import VirConv8x
    batch = scenes.make_batch_mm([2, 7], n_lidar=4096, n_virtual=6000, max_voxels=3000, training=True)
    m = VirConv8x(CFG8, 8, [1408, 1600, 80], discard_mode='paper', discard_rng='device', precision='bf16')
    fill_module(m, 667)
    m.to(DEV).train()
    state = copy.deepcopy(m.state_dict())
    res = []
    for _ in range(2):
        m.load_state_dict(state)
        for p in m.parameters():
            p.grad = None
        bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in batch.arrays.items()}
        bd.update(batch_size=2, calib=batch.calib, aug_param=torch.from_numpy(batch.aug_param),
                  stvd_seed=torch.tensor([1234], dtype=torch.int64, device=DEV))
        out = m(bd)
        pub = {f'{g}:{k}': t for g in ('multi_scale_3d_features', 'multi_scale_3d_features_mm') for k, t in out[g].items()}
        sum(t.features.mean() for t in pub.values()).backward()
        torch.cuda.synchronize()
        rec = {k: t.features.detach().clone() for k, t in pub.items()}
        rec.update({'i' + k: t.indices.clone() for k, t in pub.items()})
        rec.update({'g' + k: v.grad.clone() for k, v in m.named_parameters()})
        rec.update({'b' + k: v.clone() for k, v in m.named_buffers()})
        res.append(rec)
    for k in res[0]:
        assert torch.equal(res[0][k], res[1][k]), k


def test_module_path_raises_or_warns(lib_built, det_mode):
    from virconv_b200 import executor
    from virconv_b200.backbone import VirConvL8x
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], precision='bf16')
    fill_module(m, 666)
    m.to(DEV).train()
    batch = _batch([8, 9], n_lidar=2048, n_virtual=3000, max_voxels=2500)
    saved = executor.ENABLED
    executor.ENABLED = False
    try:
        with pytest.raises(RuntimeError, match='VIRCONV_EXECUTOR=0'):
            m(dict(batch))
        torch.use_deterministic_algorithms(True, warn_only=True)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter('always')
            m(dict(batch))
        assert any('module path' in str(x.message) for x in w)
    finally:
        executor.ENABLED = saved
    torch.use_deterministic_algorithms(True)
    m(dict(batch))          # the plan executor: no error

