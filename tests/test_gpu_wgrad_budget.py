"""The tensor-core weight gradient under a CTA budget per launch: the cap of vc_conv_wgrad_tc3_config bounds a launch's CTAs
over all its passes (blockIdx.y), not per pass.  For every multi-pass layer shape of VirConv-L, at caps 1 .. 132 and from
one row to ~40 k rows: the launch geometry keeps grid.x * passes <= cap, the result matches the float64 sum of the same
bf16-rounded operands, and the deterministic mode gives the same bits at every cap."""
import pytest
import torch

from oracle.testing import rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
# (cin, cout, K): every layer shape of VirConv-L whose wgrad runs in more than one pass
SHAPES = [(16, 32, 27), (32, 16, 27), (32, 32, 27), (64, 32, 27), (32, 64, 27), (64, 64, 27), (32, 32, 9), (64, 64, 3)]
CAPS = (1, 7, 33, 66, 132)
ROWS = (1, 129, 40000)


def _lib():
    from virconv_b200 import _lib as L
    return L, L.load()


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=DEV)


def geometry(lib, cin, cout, K, n_rows, cap):
    from virconv_b200 import _lib as L
    out = L.host_i32([0, 0])
    L.check(lib.vc_wgrad_launch_geometry(cin, cout, K, n_rows, cap, out), 'vc_wgrad_launch_geometry')
    return out[0], out[1]


def _problem(cin, cout, K, n, seed):
    """bf16-rounded operands and a neighbour table [K, n] (about a third of the entries present, the centre offset of a
    submanifold table always) over n input rows"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(n, cin, device=DEV, generator=g).to(torch.bfloat16)
    dy = torch.randn(n, cout, device=DEV, generator=g).to(torch.bfloat16)
    idx = torch.randint(0, n, (K, n), device=DEV, generator=g, dtype=torch.int32)
    keep = torch.rand(K, n, device=DEV, generator=g) < 0.35
    keep[K // 2] = True
    nbr = torch.where(keep, idx, torch.full_like(idx, -1)).contiguous()
    return x, dy, nbr


def _want(x, dy, nbr):
    """float64 dW [cout, K, cin] of the same operands"""
    K = nbr.shape[0]
    want = torch.zeros(K, x.shape[1], dy.shape[1], dtype=torch.float64, device=DEV)
    xd, dd, nl = x.double(), dy.double(), nbr.long()
    for k in range(K):
        o = torch.nonzero(nl[k] >= 0).squeeze(1)
        want[k] = xd[nl[k, o]].t() @ dd[o]
    return want.permute(2, 0, 1)


@pytest.mark.parametrize('n', ROWS)
@pytest.mark.parametrize('cin,cout,K', SHAPES)
def test_wgrad_under_cap(lib_built, cin, cout, K, n):
    from virconv_b200 import ops
    L, lib = _lib()
    err = ops.tc_error_flag(DEV)
    x, dy, nbr = _problem(cin, cout, K, n, cin * 1000 + cout * 10 + K + n)
    want = _want(x, dy, nbr)
    # the per-operator path (one CTA per SM for each pass)
    ws = _ws(lib.vc_conv_wgrad_tc_ws_bytes(n, cin, cout, K))
    dw = torch.empty(cout, K, cin, device=DEV)
    L.check(lib.vc_conv_wgrad_tc(x.data_ptr(), dy.data_ptr(), nbr.data_ptr(), dw.data_ptr(), n, cin, cout, K, ws.data_ptr(),
                                 ws.numel(), err.data_ptr(), ops._stream()), 'vc_conv_wgrad_tc')
    wsd = _ws(lib.vc_conv_wgrad_tc_det_ws_bytes(n, cin, cout, K))
    outs = []
    try:
        for cap in CAPS:
            gx, passes = geometry(lib, cin, cout, K, n, cap)
            assert gx >= 1 and passes >= 1
            if passes <= cap:
                assert gx * passes <= cap, (cap, gx, passes)
            else:
                assert gx == 1
            L.check(lib.vc_conv_wgrad_tc3_config(1, cap), 'vc_conv_wgrad_tc3_config')
            d = torch.empty(cout, K, cin, device=DEV)
            L.check(lib.vc_conv_wgrad_tc_det(x.data_ptr(), dy.data_ptr(), nbr.data_ptr(), d.data_ptr(), n, cin, cout, K,
                                             wsd.data_ptr(), wsd.numel(), err.data_ptr(), ops._stream()), 'vc_conv_wgrad_tc_det')
            outs.append(d)
    finally:
        lib.vc_conv_wgrad_tc3_config(1, 0)
    torch.cuda.synchronize()
    assert int(err.item()) == 0
    assert rel_err(dw.double(), want) < 1.6e-6
    assert rel_err(outs[0].double(), want) < 1.6e-6
    for o in outs[1:]:
        assert torch.equal(o, outs[0])

