"""GPU parity tests, operator level: every C-ABI kernel against the CPU oracle on the same seeded inputs.
Integer / index work must be bit exact; fp32 features within 1e-4 (max|d| / max|ref|, BASELINE north_star)."""
import numpy as np
import pytest
import torch

from oracle import rulebook as orb
from oracle import spconv_cpu as osp
from oracle import index2uv as ouv
from oracle.testing import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _dev():
    return torch.device('cuda:0')


def _coords(rng, n, batch, shape, unique=True):
    cols = [rng.integers(0, batch, n)] + [rng.integers(0, s, n) for s in shape]
    c = np.stack(cols, 1).astype(np.int32)
    if unique:
        c = np.unique(c, axis=0)
        rng.shuffle(c)
    return np.ascontiguousarray(c)


# ---------------------------------------------------------------------------------------------- rulebooks
@pytest.mark.parametrize('n,batch,shape', [(0, 1, [5, 6, 7]), (1, 1, [3, 3, 3]), (700, 2, [9, 10, 11]),
                                           (20000, 2, [41, 160, 141]), (3000, 3, [81, 1600, 1408])])
def test_subm3d_rulebook_bit_exact(lib_built, n, batch, shape):
    from virconv_b200 import ops
    rng = np.random.default_rng(n + 1)
    c = _coords(rng, n, batch, shape) if n else np.zeros((0, 4), np.int32)
    rb = ops.build_subm_rulebook(torch.from_numpy(c).to(_dev()), batch, shape, 3)
    want = orb.subm_rulebook(c, shape, 3)
    assert np.array_equal(rb.nbr.cpu().numpy(), want)
    assert np.array_equal(rb.pair_num.cpu().numpy(), (want >= 0).sum(1))
    pairs, num = rb.indice_pairs()
    wp, wn = orb.pairs_from_nbr(want)
    assert np.array_equal(num.cpu().numpy(), wn)
    if c.shape[0]:
        assert np.array_equal(pairs.cpu().numpy(), wp)


@pytest.mark.parametrize('n,shape', [(500, [12, 9]), (30000, [1600, 600]), (30000, [175, 75])])
def test_subm2d_rulebook_with_duplicates(lib_built, n, shape):
    from virconv_b200 import ops
    rng = np.random.default_rng(n)
    c = _coords(rng, n, 2, shape, unique=False)
    rb = ops.build_subm_rulebook(torch.from_numpy(c).to(_dev()), 2, shape, 3)
    want = orb.subm_rulebook(c, shape, 3)
    assert not rb.unique_coords
    assert np.array_equal(rb.nbr.cpu().numpy(), want)   # lowest row index wins on duplicate pixels


GEOS = [dict(ksize=3, stride=2, padding=1), dict(ksize=3, stride=2, padding=(0, 1, 1)),
        dict(ksize=(3, 1, 1), stride=(2, 1, 1), padding=0), dict(ksize=3, stride=1, padding=1),
        dict(ksize=(3, 3, 3), stride=(2, 2, 2), padding=0), dict(ksize=2, stride=2, padding=0),
        dict(ksize=3, stride=2, padding=2, dilation=(2, 3, 2)),     # dilated: marked per kernel offset
        dict(ksize=3, stride=2, padding=1, ndim=2)]                 # 2-D: the last two dimensions of `shape`


@pytest.mark.parametrize('geo', GEOS)
@pytest.mark.parametrize('n,batch,shape', [(1, 1, [5, 5, 5]), (900, 2, [9, 10, 11]), (25000, 2, [81, 400, 352])])
def test_conv_rulebook_bit_exact(lib_built, geo, n, batch, shape):
    from virconv_b200 import ops
    rng = np.random.default_rng(n)
    shape = shape[3 - geo.get('ndim', 3):]
    c = _coords(rng, n, batch, shape)
    dl = geo.get('dilation', 1)
    rb = ops.build_conv_rulebook(torch.from_numpy(c).to(_dev()), batch, shape, geo['ksize'], geo['stride'],
                                 geo['padding'], dl)
    oi, osh, nf, nb = orb.conv_rulebook(c, shape, geo['ksize'], geo['stride'], geo['padding'], dl)
    assert rb.out_shape == osh
    assert np.array_equal(rb.out_indices.cpu().numpy(), oi)           # ascending linear index, batch major
    assert np.array_equal(rb.nbr.cpu().numpy(), nf)
    assert np.array_equal(rb.nbr_bwd.cpu().numpy(), nb)
    assert np.array_equal(rb.pair_num.cpu().numpy(), (nf >= 0).sum(1))
    assert np.all(np.diff(rb.out_indices[:, 0].cpu().numpy()) >= 0)   # batch-contiguous rows (SURVEY a15)


def test_virconv_shape_chain(lib_built):
    """z 81->41->21->10->4, y 1600->800->400->200, x 1408->704->352->176 (SURVEY §4)."""
    from virconv_b200 import _lib
    lib = _lib.load()
    shape = [81, 1600, 1408]
    for pad in [(1, 1, 1), (1, 1, 1), (0, 1, 1)]:
        o = _lib.host_i32([0, 0, 0])
        assert lib.vc_conv_out_shape(3, _lib.host_i32(shape), _lib.host_i32([3, 3, 3]), _lib.host_i32([2, 2, 2]),
                                     _lib.host_i32(pad), _lib.host_i32([1, 1, 1]), o) == 0
        shape = list(o)
    assert shape == [10, 200, 176]
    o = _lib.host_i32([0, 0, 0])
    lib.vc_conv_out_shape(3, _lib.host_i32(shape), _lib.host_i32([3, 1, 1]), _lib.host_i32([2, 1, 1]),
                          _lib.host_i32([0, 0, 0]), _lib.host_i32([1, 1, 1]), o)
    assert list(o) == [4, 200, 176]


# ---------------------------------------------------------------------------------------------- convolution
CH = [(8, 8), (16, 16), (16, 32), (32, 16), (32, 32), (32, 64), (64, 32), (64, 64), (8, 16), (64, 8)]


def _oracle_conv(feats, weight, nbr, n_out, subm, dout):
    f = feats.clone().requires_grad_(True)
    w = weight.clone().requires_grad_(True)
    out = osp.native_conv(f, w.reshape(w.shape[0], -1, w.shape[-1]), torch.from_numpy(nbr).long(), n_out, subm)
    out.backward(dout)
    return out.detach(), f.grad, w.grad


@pytest.mark.parametrize('cin,cout', CH)
def test_subm3d_conv_fwd_bwd(lib_built, cin, cout):
    from virconv_b200 import ops
    rng = np.random.default_rng(cin * 100 + cout)
    shape = [12, 40, 40]
    c = _coords(rng, 6000, 2, shape)
    n = c.shape[0]
    torch.manual_seed(cin + cout)
    feats = torch.randn(n, cin)
    weight = torch.randn(cout, 3, 3, 3, cin) * 0.1
    dout = torch.randn(n, cout)
    rb = ops.build_subm_rulebook(torch.from_numpy(c).to(_dev()), 2, shape, 3)
    f = feats.to(_dev()).requires_grad_(True)
    w = weight.to(_dev()).requires_grad_(True)
    out = ops.SparseConvFn.apply(f, w, rb)
    out.backward(dout.to(_dev()))
    ro, rdf, rdw = _oracle_conv(feats, weight, orb.subm_rulebook(c, shape, 3), n, True, dout)
    assert rel_err(out.detach().cpu(), ro) < TOL
    assert rel_err(f.grad.cpu(), rdf) < TOL
    assert rel_err(w.grad.cpu(), rdw) < TOL


@pytest.mark.parametrize('cin,cout', [(16, 32), (32, 64), (64, 64), (8, 8)])
@pytest.mark.parametrize('geo', GEOS[:3])
def test_strided_conv_fwd_bwd(lib_built, cin, cout, geo):
    from virconv_b200 import ops
    rng = np.random.default_rng(cin + cout)
    shape = [21, 40, 36]
    c = _coords(rng, 5000, 2, shape)
    n = c.shape[0]
    torch.manual_seed(1)
    ks = geo['ksize'] if isinstance(geo['ksize'], tuple) else (geo['ksize'],) * 3
    feats = torch.randn(n, cin)
    weight = torch.randn(cout, *ks, cin) * 0.1
    rb = ops.build_conv_rulebook(torch.from_numpy(c).to(_dev()), 2, shape, geo['ksize'], geo['stride'], geo['padding'])
    oi, osh, nf, nb = orb.conv_rulebook(c, shape, geo['ksize'], geo['stride'], geo['padding'])
    dout = torch.randn(oi.shape[0], cout)
    f = feats.to(_dev()).requires_grad_(True)
    w = weight.to(_dev()).requires_grad_(True)
    out = ops.SparseConvFn.apply(f, w, rb)
    out.backward(dout.to(_dev()))
    ro, rdf, rdw = _oracle_conv(feats, weight, nf, oi.shape[0], False, dout)
    assert rel_err(out.detach().cpu(), ro) < TOL
    assert rel_err(f.grad.cpu(), rdf) < TOL
    assert rel_err(w.grad.cpu(), rdw) < TOL


@pytest.mark.parametrize('c', [8, 16, 32])
def test_subm2d_conv_duplicates_fwd_bwd(lib_built, c):
    """image branch: many rows per pixel; dgrad goes through the scatter kernel."""
    from virconv_b200 import ops
    rng = np.random.default_rng(c)
    shape = [60, 40]
    co = _coords(rng, 7000, 2, shape, unique=False)
    n = co.shape[0]
    torch.manual_seed(c)
    feats, weight, dout = torch.randn(n, c), torch.randn(c, 3, 3, c) * 0.1, torch.randn(n, c)
    rb = ops.build_subm_rulebook(torch.from_numpy(co).to(_dev()), 2, shape, 3)
    f = feats.to(_dev()).requires_grad_(True)
    w = weight.to(_dev()).requires_grad_(True)
    out = ops.SparseConvFn.apply(f, w, rb)
    out.backward(dout.to(_dev()))
    ro, rdf, rdw = _oracle_conv(feats, weight, orb.subm_rulebook(co, shape, 3), n, True, dout)
    assert rel_err(out.detach().cpu(), ro) < TOL
    assert rel_err(f.grad.cpu(), rdf) < TOL
    assert rel_err(w.grad.cpu(), rdw) < TOL


def test_conv_against_dense_conv3d(lib_built):
    """Ground truth independent of the oracle: brute-force dense torch conv3d on a tiny grid."""
    import torch.nn.functional as F
    from virconv_b200 import spconv_compat as sp
    rng = np.random.default_rng(3)
    shape, B = [9, 10, 11], 2
    c = _coords(rng, 500, B, shape)
    feats = torch.randn(c.shape[0], 16)
    x = sp.SparseConvTensor(feats.to(_dev()), torch.from_numpy(c).to(_dev()), shape, B)
    dense_in = x.dense().cpu()
    for cls, kw, dkw in [(sp.SubMConv3d, dict(kernel_size=3), dict(padding=1)),
                         (sp.SparseConv3d, dict(kernel_size=3, stride=2, padding=1), dict(stride=2, padding=1)),
                         (sp.SparseConv3d, dict(kernel_size=(3, 1, 1), stride=(2, 1, 1), padding=0),
                          dict(stride=(2, 1, 1), padding=0))]:
        m = cls(16, 32, bias=False, **kw).to(_dev())
        y = m(x)
        ref = F.conv3d(dense_in, m.weight.detach().cpu().permute(0, 4, 1, 2, 3), **dkw)
        if m.subm:
            got = y.features.detach().cpu()
            want = ref[c[:, 0], :, c[:, 1], c[:, 2], c[:, 3]]
            assert rel_err(got, want) < TOL
        else:
            assert list(y.dense().shape) == list(ref.shape)
            assert rel_err(y.dense().detach().cpu(), ref) < TOL


def test_empty_and_tail_tiles(lib_built):
    from virconv_b200 import ops
    shape = [5, 6, 7]
    for n in (1, 127, 128, 129):
        rng = np.random.default_rng(n)
        c = _coords(rng, n, 1, shape)
        rb = ops.build_subm_rulebook(torch.from_numpy(c).to(_dev()), 1, shape, 3)
        feats, weight = torch.randn(c.shape[0], 8), torch.randn(16, 3, 3, 3, 8)
        out = ops.conv_forward(feats.to(_dev()), weight.to(_dev()), rb)
        ro = osp.native_conv(feats, weight.reshape(16, 27, 8), torch.from_numpy(orb.subm_rulebook(c, shape, 3)).long(),
                             c.shape[0], True)
        assert rel_err(out.cpu(), ro) < TOL


# ---------------------------------------------------------------------------------------------- BN + ReLU
@pytest.mark.parametrize('training', [True, False])
@pytest.mark.parametrize('cin,cout', [(8, 8), (32, 16), (64, 64)])
def test_conv_bn_relu_fused(lib_built, training, cin, cout):
    from virconv_b200 import ops
    rng = np.random.default_rng(5)
    shape = [12, 30, 30]
    c = _coords(rng, 5000, 2, shape)
    n = c.shape[0]
    torch.manual_seed(0)
    feats, weight, dy = torch.randn(n, cin), torch.randn(cout, 3, 3, 3, cin) * 0.1, torch.randn(n, cout)
    bn = torch.nn.BatchNorm1d(cout, eps=1e-3, momentum=0.01)
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_(0, 0.1)
        bn.running_mean.normal_(0, 0.1)
        bn.running_var.uniform_(0.5, 1.5)
    bn.train(training)
    import copy
    bn_g = copy.deepcopy(bn).to(_dev())
    fr = feats.clone().requires_grad_(True)
    wr = weight.clone().requires_grad_(True)
    xr = osp.native_conv(fr, wr.reshape(cout, 27, cin), torch.from_numpy(orb.subm_rulebook(c, shape, 3)).long(), n, True)
    pre = bn(xr)
    yr = torch.relu(pre)
    # a pre-activation within rounding distance of 0 may take the other ReLU branch on the GPU; keep those
    # (a handful of) elements out of the gradient comparison instead of loosening the tolerance
    dy = dy * (pre.detach().abs() > 1e-4)
    yr.backward(dy)
    rb = ops.build_subm_rulebook(torch.from_numpy(c).to(_dev()), 2, shape, 3)
    f = feats.to(_dev()).requires_grad_(True)
    w = weight.to(_dev()).requires_grad_(True)
    y = ops.ConvBNReLUFn.apply(f, w, bn_g.weight, bn_g.bias, bn_g.running_mean, bn_g.running_var, rb, training, 1e-3,
                               0.01)
    y.backward(dy.to(_dev()))
    assert rel_err(y.detach().cpu(), yr.detach()) < TOL
    assert rel_err(f.grad.cpu(), fr.grad) < 5e-4
    assert rel_err(w.grad.cpu(), wr.grad) < 5e-4
    assert rel_err(bn_g.weight.grad.cpu(), bn.weight.grad) < 5e-4
    assert rel_err(bn_g.bias.grad.cpu(), bn.bias.grad) < 5e-4
    assert rel_err(bn_g.running_mean.cpu(), bn.running_mean) < 1e-5
    assert rel_err(bn_g.running_var.cpu(), bn.running_var) < 1e-5


# ---------------------------------------------------------------------------------------------- index2uv
def test_index2uv_bit_exact_and_golden(lib_built):
    import os
    from virconv_b200 import ops, scenes
    g = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'index2uv.npz'))
    for ci in range(int(g['n_cases'])):
        idx, want, stride, aug = g[f'idx{ci}'], g[f'uv{ci}'], int(g[f'stride{ci}']), g[f'aug{ci}']
        aug = aug if aug.shape[0] else None
        calibs = [scenes.Calib(), scenes.Calib()]
        params = ops.projection_params(calibs, aug, 2, _dev())
        uv = ops.index2uv(torch.from_numpy(idx).to(_dev()), 2, params, stride).cpu().numpy()
        assert np.array_equal(uv, ouv.index2uv(idx, 2, calibs, stride, aug))   # oracle: bit exact
        assert np.array_equal(uv, want)                                        # the reference's own output


def test_index2uv_edge_cases(lib_built):
    """voxels behind / at the camera plane: inf, NaN and negative pixel coordinates must clamp like the oracle."""
    from virconv_b200 import ops, scenes
    rng = np.random.default_rng(0)
    idx = np.stack([rng.integers(0, 2, 4000), rng.integers(0, 81, 4000), rng.integers(0, 1600, 4000),
                    rng.integers(0, 12, 4000)], 1).astype(np.int32)        # x < 0.6 m: rect z around 0
    calibs = [scenes.Calib(), scenes.Calib()]
    aug = np.array([[0.7, 1, 0.95], [-0.7, 0, 1.05]], np.float32)
    for stride in (1, 8):
        params = ops.projection_params(calibs, aug, 2, _dev())
        uv = ops.index2uv(torch.from_numpy(idx).to(_dev()), 2, params, stride).cpu().numpy()
        assert np.array_equal(uv, ouv.index2uv(idx, 2, calibs, stride, aug))


# ---------------------------------------------------------------------------------------------- dense / gather
def test_dense_and_gather(lib_built):
    from virconv_b200 import ops, spconv_compat as sp
    rng = np.random.default_rng(1)
    shape = [4, 20, 17]
    c = _coords(rng, 900, 2, shape)
    feats = torch.randn(c.shape[0], 64)
    x = sp.SparseConvTensor(feats.to(_dev()).requires_grad_(True), torch.from_numpy(c).to(_dev()), shape, 2)
    d = x.dense()
    ref = osp.SparseConvTensor(feats, torch.from_numpy(c), shape, 2).dense()
    assert torch.equal(d.detach().cpu(), ref)
    n, cc, dd, h, w = d.shape
    assert d.view(n, cc * dd, h, w).shape == (2, 256, 20, 17)          # height_compression.py:30-31
    g = torch.randn_like(d)
    d.backward(g)
    want = g.cpu()[c[:, 0], :, c[:, 1], c[:, 2], c[:, 3]]
    assert torch.equal(x.features.grad.cpu(), want)
    rows = torch.from_numpy(np.sort(rng.permutation(c.shape[0])[:500]).astype(np.int32)).to(_dev())
    assert torch.equal(ops.gather_rows(feats.to(_dev()), rows).cpu(), feats[rows.cpu().long()])
    idx = torch.from_numpy(c).to(_dev())
    assert torch.equal(ops.gather_rows(idx, rows).cpu(), torch.from_numpy(c)[rows.cpu().long()])


# ---------------------------------------------------------------------------------------------- tensor cores
def _bf(t):
    return t.bfloat16().float()


@pytest.mark.parametrize('cin,cout', [(8, 8), (16, 16), (32, 16), (16, 32), (32, 32), (64, 32), (32, 64), (64, 64), (16, 64), (64, 16)])
def test_tc_subm3d_conv_fwd_dgrad(lib_built, cin, cout):
    """tensor-core path: exact-operand check (oracle fed the same bf16-rounded operands, fp32 accumulate) at 1e-4, and
    the bf16-precision check against the full-fp32 oracle at 2e-2; pipeline-timeout flag must stay 0."""
    from virconv_b200 import ops
    rng = np.random.default_rng(cin * 100 + cout)
    shape = [12, 40, 40]
    c = _coords(rng, 9000, 2, shape)
    n = c.shape[0]
    torch.manual_seed(cin + cout)
    feats, weight, dout = torch.randn(n, cin), torch.randn(cout, 3, 3, 3, cin) * 0.1, torch.randn(n, cout)
    rb = ops.build_subm_rulebook(torch.from_numpy(c).to(_dev()), 2, shape, 3)
    f = feats.to(_dev()).requires_grad_(True)
    w = weight.to(_dev()).requires_grad_(True)
    out = ops.SparseConvFn.apply(f, w, rb, 'bf16')
    out.backward(dout.to(_dev()))
    torch.cuda.synchronize()
    assert int(ops.tc_error_flag(_dev()).item()) == 0
    nbr = orb.subm_rulebook(c, shape, 3)
    ro, _, _ = _oracle_conv(_bf(feats), _bf(weight), nbr, n, True, dout)
    assert rel_err(out.detach().cpu(), ro) < TOL
    _, rdf, _ = _oracle_conv(feats, _bf(weight), nbr, n, True, _bf(dout))       # dgrad gathers bf16(dout)
    assert rel_err(f.grad.cpu(), rdf) < TOL
    _, _, rdw = _oracle_conv(_bf(feats), weight, nbr, n, True, _bf(dout))        # wgrad: both operands bf16
    assert rel_err(w.grad.cpu(), rdw) < TOL
    ro32, rdf32, rdw32 = _oracle_conv(feats, weight, nbr, n, True, dout)
    assert rel_err(out.detach().cpu(), ro32) < 2e-2
    assert rel_err(f.grad.cpu(), rdf32) < 2e-2
    assert rel_err(w.grad.cpu(), rdw32) < 2e-2


@pytest.mark.parametrize('cin,cout', [(16, 32), (32, 64), (64, 64)])
@pytest.mark.parametrize('geo', GEOS[:3])
def test_tc_strided_conv_fwd_dgrad(lib_built, cin, cout, geo):
    from virconv_b200 import ops
    rng = np.random.default_rng(cin + cout)
    shape = [21, 40, 36]
    c = _coords(rng, 5000, 2, shape)
    n = c.shape[0]
    torch.manual_seed(1)
    ks = geo['ksize'] if isinstance(geo['ksize'], tuple) else (geo['ksize'],) * 3
    feats, weight = torch.randn(n, cin), torch.randn(cout, *ks, cin) * 0.1
    rb = ops.build_conv_rulebook(torch.from_numpy(c).to(_dev()), 2, shape, geo['ksize'], geo['stride'], geo['padding'])
    oi, osh, nf, nb = orb.conv_rulebook(c, shape, geo['ksize'], geo['stride'], geo['padding'])
    dout = torch.randn(oi.shape[0], cout)
    f = feats.to(_dev()).requires_grad_(True)
    w = weight.to(_dev()).requires_grad_(True)
    out = ops.SparseConvFn.apply(f, w, rb, 'bf16')
    out.backward(dout.to(_dev()))
    torch.cuda.synchronize()
    assert int(ops.tc_error_flag(_dev()).item()) == 0
    ro, _, _ = _oracle_conv(_bf(feats), _bf(weight), nf, oi.shape[0], False, dout)
    assert rel_err(out.detach().cpu(), ro) < TOL
    _, rdf, _ = _oracle_conv(feats, _bf(weight), nf, oi.shape[0], False, _bf(dout))
    assert rel_err(f.grad.cpu(), rdf) < TOL
    _, _, rdw = _oracle_conv(_bf(feats), weight, nf, oi.shape[0], False, _bf(dout))
    assert rel_err(w.grad.cpu(), rdw) < TOL


@pytest.mark.parametrize('ctas', [1, 2])
def test_tc2_one_and_two_ctas_per_sm(lib_built, ctas):
    """The persistent conv kernel in both of its shared-memory plans (vc_conv_tc2_config: one CTA with the whole SM, two CTAs
    with half each — automatic choice elsewhere): forward, gather dgrad of a submanifold conv and the offset-scanning dgrad of a
    strided conv against the oracle fed the same bf16-rounded operands."""
    from virconv_b200 import _lib, ops
    lib = _lib.load()
    _lib.check(lib.vc_conv_tc2_config(ctas), 'vc_conv_tc2_config')
    try:
        rng = np.random.default_rng(77 + ctas)
        shape = [21, 40, 36]
        c = _coords(rng, 6000, 2, shape)
        n = c.shape[0]
        torch.manual_seed(5)
        for cin, cout, strided in ((32, 32, False), (16, 32, True), (64, 64, True)):
            if strided:
                rb = ops.build_conv_rulebook(torch.from_numpy(c).to(_dev()), 2, shape, 3, 2, 1)
                oi, _, nf, _ = orb.conv_rulebook(c, shape, 3, 2, 1)
                nbr, n_out = nf, oi.shape[0]
            else:
                rb = ops.build_subm_rulebook(torch.from_numpy(c).to(_dev()), 2, shape, 3)
                nbr, n_out = orb.subm_rulebook(c, shape, 3), n
            feats, weight, dout = torch.randn(n, cin), torch.randn(cout, 3, 3, 3, cin) * 0.1, torch.randn(n_out, cout)
            f = feats.to(_dev()).requires_grad_(True)
            w = weight.to(_dev()).requires_grad_(True)
            out = ops.SparseConvFn.apply(f, w, rb, 'bf16')
            out.backward(dout.to(_dev()))
            torch.cuda.synchronize()
            assert int(ops.tc_error_flag(_dev()).item()) == 0
            ro, _, _ = _oracle_conv(_bf(feats), _bf(weight), nbr, n_out, not strided, dout)
            assert rel_err(out.detach().cpu(), ro) < TOL, (cin, cout, strided)
            _, rdf, _ = _oracle_conv(feats, _bf(weight), nbr, n_out, not strided, _bf(dout))
            assert rel_err(f.grad.cpu(), rdf) < TOL, (cin, cout, strided)
    finally:
        _lib.check(lib.vc_conv_tc2_config(0), 'vc_conv_tc2_config')


def test_tc_subm2d_duplicates_and_tails(lib_built):
    """image-branch table (forward and the scatter-form dgrad on tensor cores) + ragged tiles"""
    from virconv_b200 import ops
    for n_req, cch in ((1, 16), (127, 32), (129, 32), (5000, 32)):
        rng = np.random.default_rng(n_req)
        shape = [60, 40]
        co = _coords(rng, n_req, 2, shape, unique=False)
        n = co.shape[0]
        torch.manual_seed(n_req)
        feats, weight, dout = torch.randn(n, cch), torch.randn(cch, 3, 3, cch) * 0.1, torch.randn(n, cch)
        rb = ops.build_subm_rulebook(torch.from_numpy(co).to(_dev()), 2, shape, 3)
        f = feats.to(_dev()).requires_grad_(True)
        w = weight.to(_dev()).requires_grad_(True)
        out = ops.SparseConvFn.apply(f, w, rb, 'bf16')
        out.backward(dout.to(_dev()))
        torch.cuda.synchronize()
        assert int(ops.tc_error_flag(_dev()).item()) == 0
        nbr = orb.subm_rulebook(co, shape, 3)
        ro, _, _ = _oracle_conv(_bf(feats), _bf(weight), nbr, n, True, dout)
        assert rel_err(out.detach().cpu(), ro) < TOL
        _, rdf, _ = _oracle_conv(feats, _bf(weight), nbr, n, True, _bf(dout))       # scatter dgrad: bf16 operands
        assert rel_err(f.grad.cpu(), rdf) < TOL
        _, _, rdw = _oracle_conv(_bf(feats), weight, nbr, n, True, _bf(dout))
        assert rel_err(w.grad.cpu(), rdw) < TOL
        _, rdf32, _ = _oracle_conv(feats, weight, nbr, n, True, dout)
        assert rel_err(f.grad.cpu(), rdf32) < 2e-2


def test_tc_backbone_bf16_vs_fp32_oracle(lib_built):
    """whole VirConv-L backbone in bf16 tensor-core mode against the fp32 oracle at a bf16 tolerance"""
    from virconv_b200 import scenes, ops
    from virconv_b200.backbone import VirConvL8x
    from oracle.backbone import VirConvL8x as OracleL
    from oracle.testing import fill_module
    cfg = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
    batch = scenes.make_batch([0, 5], n_lidar=4096, n_virtual=6000, max_voxels=6000, training=True)
    m = VirConvL8x(cfg, 8, [1408, 1600, 80], precision='bf16')
    fill_module(m, 666)
    ref = OracleL()
    ref.load_state_dict(m.state_dict())
    m.to(_dev()).train()
    ref.train()
    bd = {'voxel_features': torch.from_numpy(batch.voxel_features.copy()).to(_dev()),
          'voxel_coords': torch.from_numpy(batch.voxel_coords.copy()).to(_dev()), 'batch_size': 2, 'calib': batch.calib,
          'aug_param': batch.aug_param}
    out = m(bd)
    o = ref(torch.from_numpy(batch.voxel_features.copy()), torch.from_numpy(batch.voxel_coords.copy()), 2, batch.calib,
            batch.aug_param)
    named = dict(out['multi_scale_3d_features'])
    named['out'] = out['encoded_spconv_tensor']
    for k, t in named.items():
        assert np.array_equal(t.indices.cpu().numpy(), o[k].indices.numpy()), k     # index work stays bit exact
        e = rel_err(t.features.detach().cpu(), o[k].features.detach())
        assert e < 5e-2, (k, e)
    sum(t.features.mean() for t in named.values()).backward()
    torch.cuda.synchronize()
    assert int(ops.tc_error_flag(_dev()).item()) == 0
    assert all(torch.isfinite(p.grad).all() for p in m.parameters())


# ---------------------------------------------------------------------------------------------- voxelise + VFE
@pytest.mark.parametrize('n_virtual,max_voxels,model', [(0, 40000, 'max'), (20000, 3000, 'max'), (20000, 40000, None)])
def test_gpu_voxelize_mean_matches_first_come_reference(lib_built, n_virtual, max_voxels, model):
    """bit-exact against the numpy restatement of Point2VoxelCPU3d + MeanVFE (itself pinned by tests/golden/mean_vfe.npz)"""
    from virconv_b200 import ops, scenes
    pts_all, want = [], []
    for b, sid in enumerate([3, 4, 9]):
        p = scenes.mask_points_by_range(scenes.make_points(sid, 4096, n_virtual))
        if b == 1:
            p = np.concatenate([p, p[:500], p[:500], p[:500], p[:500], p[:500], p[:500]])   # voxels with > 5 points
            p[100:110, 2] = 5.0                                                             # z outside the range
        vox, coords, num = scenes.voxelize_first_come(p, max_voxels=max_voxels)
        want.append((scenes.mean_vfe(vox, num, model), np.concatenate([np.full((coords.shape[0], 1), b, np.int32), coords], 1),
                     num, vox))
        pts_all.append(np.concatenate([np.full((p.shape[0], 1), b, np.float32), p], 1))
    pts = torch.from_numpy(np.concatenate(pts_all)).to(_dev())
    f, c, nm, v = ops.voxelize_mean(pts, 3, max_voxels=max_voxels, vfe_model=model, want_voxels=True)
    wf, wc, wn, wv = (np.concatenate([w[i] for w in want]) for i in range(4))
    assert np.array_equal(c.cpu().numpy(), wc)
    assert np.array_equal(nm.cpu().numpy(), wn)
    assert np.array_equal(v.cpu().numpy(), wv)
    assert np.array_equal(f.cpu().numpy(), wf)


def test_gpu_voxelize_golden_and_empty_sample(lib_built):
    import os
    from virconv_b200 import ops
    g = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'mean_vfe.npz'))
    # rebuild a point list from the golden voxels (point order = voxel-major): voxelising it again must give the same voxels
    vox, num = g['voxels'], g['num']
    pts = np.concatenate([vox[i, :num[i]] for i in range(vox.shape[0])])
    pts = np.concatenate([np.full((pts.shape[0], 1), 1, np.float32), pts], 1)          # only sample 1 has points
    f, c, nm = ops.voxelize_mean(torch.from_numpy(pts).to(_dev()), 2, max_voxels=3000, vfe_model='max')
    assert np.array_equal(f.cpu().numpy(), g['features'])                               # the reference MeanVFE's output
    assert np.array_equal(c.cpu().numpy()[:, 1:], g['coords']) and np.all(c.cpu().numpy()[:, 0] == 1)
    assert np.array_equal(nm.cpu().numpy(), num)


def test_voxel2pinds(lib_built):
    from virconv_b200 import ops
    rng = np.random.default_rng(2)
    shape = [10, 20, 18]
    c = _coords(rng, 700, 2, shape)
    got = ops.voxel2pinds(torch.from_numpy(c).to(_dev()), 2, shape).cpu().numpy()
    want = -np.ones([2] + shape, np.int32)
    want[c[:, 0], c[:, 1], c[:, 2], c[:, 3]] = np.arange(c.shape[0])
    assert np.array_equal(got, want)
