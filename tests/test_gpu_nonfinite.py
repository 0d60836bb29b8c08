"""NaN and +-Inf through the training step's kernels, against the operations they replace run in float64 on the kernels' own
operands (bf16-rounded where a kernel reads bf16).  For every output, isfinite(got) equals isfinite(ref) element by element
(the kind of non-finite value is not compared), and the elements finite in both meet the tolerance the kernel's own test
uses.  Backward references come from autograd: torch's ReLU backward passes the gradient wherever the activation is not
<= 0, NaN included.

Covered: the conv forward / dgrad / wgrad (bf16 tensor-core and fp32, submanifold, strided and many-to-one 2-D tables,
normal and deterministic; NaN beside a column-slice input and past a device row count), BatchNorm + ReLU forward (fused
into the conv and not) and backward, the fused voxel-RoI pooling, masked_mean, the voxeliser (eager and captured), whole
VirConv-L / VirConv-T training steps whose guarded update has to skip a poisoned batch, and the captured eval forward
(GraphedForward) against the float64 module path."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import audit
from oracle.testing import fill_module

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
NAN, INF = float('nan'), float('inf')
N = 128 * 5 + 37                     # five whole 128-row tiles and a ragged sixth
SHAPE3 = [6, 40, 40]
SHAPE2 = [30, 40]
CFG_L = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG_T = dict(CFG_L, LAYER_DISCARD_RATE=0.15, MM=True)


def _lib():
    from virconv_b200 import _lib as L
    return L, L.load()


def _err():
    from virconv_b200 import ops
    return ops.tc_error_flag(DEV)


def _st():
    from virconv_b200 import ops
    return ops._stream()


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=DEV)


@pytest.fixture(autouse=True)
def _built(lib_built):
    yield
    torch.cuda.synchronize()
    assert int(_err().item()) == 0


@pytest.fixture(params=[1, 2], ids=['1cta', '2cta'])
def ctas(request):
    L, lib = _lib()
    L.check(lib.vc_conv_tc2_config(request.param), 'vc_conv_tc2_config')
    try:
        yield request.param
    finally:
        lib.vc_conv_tc2_config(0)


def match(got, ref, tol, where):
    """isfinite(got) == isfinite(ref) everywhere; max|got - ref| / max|ref| < tol over the elements finite in both"""
    got, ref = torch.as_tensor(got).detach().double().cpu(), torch.as_tensor(ref).detach().double().cpu()
    assert got.shape == ref.shape, (where, got.shape, ref.shape)
    fg, fr = torch.isfinite(got), torch.isfinite(ref)
    bad = (fg != fr).nonzero()
    assert bad.shape[0] == 0, (where, 'finiteness differs at', bad[:5].tolist(), int(bad.shape[0]),
                               got[tuple(bad[0])].item(), ref[tuple(bad[0])].item())
    if fr.any():
        e = float((got[fr] - ref[fr]).abs().max() / ref[fr].abs().max().clamp_min(1e-30))
        assert e < tol, (where, e, tol)


def _weights(ci, co, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(co, K, ci, device=DEV, generator=g) * (2.0 / (K * ci)) ** 0.5).contiguous()


def _poisoned(n, c, seed, rows, dtype=torch.float32):
    """randn [n, c] with a NaN row and a +Inf row at rows = (r_nan, r_inf)"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    t = torch.randn(n, c, device=DEV, generator=g)
    t[rows[0]] = NAN
    t[rows[1]] = INF
    return t.to(dtype)


# ------------------------------------------------------------------------------------------------ conv tables
def _coords3(n, seed):
    rng = np.random.default_rng(seed)
    cells = rng.choice(2 * SHAPE3[0] * SHAPE3[1] * SHAPE3[2] // 4, size=n, replace=False)
    b, r = np.divmod(cells, SHAPE3[0] * SHAPE3[1] * SHAPE3[2] // 4)
    z, r = np.divmod(r, SHAPE3[1] * SHAPE3[2] // 4)
    y, x = np.divmod(r, SHAPE3[2] // 4)
    return torch.from_numpy(np.stack([b, z, y, x], 1).astype(np.int32)).to(DEV)


def _table(kind):
    """-> dict(nbr [K, n_out], n_in, n_out, K, and per kind the dgrad's table)"""
    from virconv_b200 import ops
    co = _coords3(N, 21)
    if kind == 'subm3d':
        nbr = ops.build_subm_rulebook(co, 2, SHAPE3, 3).nbr
        return dict(nbr=nbr, n_in=N, n_out=N, K=27, dgrad=('gather', nbr, 1))
    if kind == 'strided':
        rb = ops.build_conv_rulebook(co, 2, SHAPE3, 3, 2, 1)
        return dict(nbr=rb.nbr, n_in=N, n_out=rb.n_out, K=27, dgrad=('gather', rb.nbr_bwd, 0))
    nbr, rep = _table2d(N)
    return dict(nbr=nbr, n_in=N, n_out=N, K=9, dgrad=('2d', nbr, rep))


def _table2d(rows):
    """many-to-one 2-D table over the first `rows` of N rows (~40 % of them on 12 hot pixels), padded to N rows as a
    capacity-sized table: nbr tail -1, rep tail = the row itself"""
    L, lib = _lib()
    rng = np.random.default_rng(22)
    hot = rng.integers(0, 2 * SHAPE2[0] * SHAPE2[1], 12)
    pix = np.where(rng.random(N) < 0.6, rng.integers(0, 2 * SHAPE2[0] * SHAPE2[1], N), hot[rng.integers(0, 12, N)])[:rows]
    b, r = np.divmod(pix, SHAPE2[0] * SHAPE2[1])
    v, u = np.divmod(r, SHAPE2[1])
    ci = torch.from_numpy(np.stack([b, v, u], 1).astype(np.int32)).to(DEV)
    nbr = torch.full((9, N), -1, dtype=torch.int32, device=DEV)
    nb = torch.empty(9, rows, dtype=torch.int32, device=DEV)
    pn = torch.empty(9, dtype=torch.int32, device=DEV)
    rep = torch.arange(N, dtype=torch.int32, device=DEV)
    rp = torch.empty(rows, dtype=torch.int32, device=DEV)
    ws = _ws(lib.vc_subm_rulebook_ws_bytes(rows))
    L.check(lib.vc_subm_rulebook_rep(ci.data_ptr(), rows, 2, 2, L.host_i32(SHAPE2), L.host_i32([3, 3]), L.host_i32([1, 1]), nb.data_ptr(),
                                     pn.data_ptr(), rp.data_ptr(), ws.data_ptr(), ws.numel(), _st()), 'vc_subm_rulebook_rep')
    nbr[:, :rows] = nb
    rep[:rows] = rp
    return nbr, rep


def _conv_fwd(prec, det, x, w, nbr, n_out, ci, co, K):
    L, lib = _lib()
    out = torch.full((n_out, co), 7.0, device=DEV)
    if det:
        ws = _ws(lib.vc_conv_fwd_det_ws_bytes(n_out, ci, co, K))
        sums = torch.empty(2, co, dtype=torch.float64, device=DEV)
        L.check(lib.vc_conv_fwd_det(int(prec == 'bf16'), x.data_ptr(), w.data_ptr(), nbr.data_ptr(), out.data_ptr(), n_out, ci, co, K,
                                    sums.data_ptr(), ws.data_ptr(), ws.numel(), _err().data_ptr(), _st()), 'vc_conv_fwd_det')
    elif prec == 'bf16':
        ws = _ws(lib.vc_conv_tc_ws_bytes(ci, co, K))
        L.check(lib.vc_conv_fwd_tc(x.data_ptr(), w.data_ptr(), nbr.data_ptr(), out.data_ptr(), n_out, ci, co, K, None, ws.data_ptr(),
                                   ws.numel(), _err().data_ptr(), _st()), 'vc_conv_fwd_tc')
    else:
        ws = _ws(lib.vc_conv_ws_bytes(ci, co, K))
        L.check(lib.vc_conv_fwd_f32(x.data_ptr(), w.data_ptr(), nbr.data_ptr(), out.data_ptr(), n_out, ci, co, K, None, ws.data_ptr(),
                                    ws.numel(), _st()), 'vc_conv_fwd_f32')
    return out


def _conv_dgrad(prec, form, dout, w, t, ci, co):
    L, lib = _lib()
    K, n = t['K'], t['n_in']
    tc = prec == 'bf16'
    if form == 'scatter':
        din = torch.zeros(n, ci, device=DEV)
        ws = _ws(lib.vc_conv_tc_ws_bytes(ci, co, K) if tc else lib.vc_conv_ws_bytes(ci, co, K))
        if tc:
            L.check(lib.vc_conv_dgrad_scatter_tc(dout.data_ptr(), w.data_ptr(), t['nbr'].data_ptr(), din.data_ptr(), t['n_out'], ci, co, K,
                                                 ws.data_ptr(), ws.numel(), _err().data_ptr(), _st()), 'vc_conv_dgrad_scatter_tc')
        else:
            L.check(lib.vc_conv_dgrad_scatter_f32(dout.data_ptr(), w.data_ptr(), t['nbr'].data_ptr(), din.data_ptr(), t['n_out'], ci, co,
                                                  K, ws.data_ptr(), ws.numel(), _st()), 'vc_conv_dgrad_scatter_f32')
        return din
    din = torch.full((n, ci), 7.0, device=DEV)
    if form == '2d':
        rep = t['dgrad'][2]
        ws = _ws(lib.vc_conv_dgrad_gather2d_ws_bytes(n, ci, co, K))
        fn = lib.vc_conv_dgrad_gather2d_tc if tc else lib.vc_conv_dgrad_gather2d_f32
        args = (dout.data_ptr(), w.data_ptr(), t['nbr'].data_ptr(), rep.data_ptr(), din.data_ptr(), n, None, ci, co, K, ws.data_ptr(),
                ws.numel()) + ((_err().data_ptr(),) if tc else ()) + (_st(),)
        L.check(fn(*args), 'gather2d dgrad')
        return din
    _, nbr_t, mirror = t['dgrad']
    ws = _ws(lib.vc_conv_tc_ws_bytes(ci, co, K) if tc else lib.vc_conv_ws_bytes(ci, co, K))
    if tc:
        L.check(lib.vc_conv_dgrad_tc(dout.data_ptr(), w.data_ptr(), nbr_t.data_ptr(), din.data_ptr(), n, ci, co, K, mirror, ws.data_ptr(),
                                     ws.numel(), _err().data_ptr(), _st()), 'vc_conv_dgrad_tc')
    else:
        L.check(lib.vc_conv_dgrad_f32(dout.data_ptr(), w.data_ptr(), nbr_t.data_ptr(), din.data_ptr(), n, ci, co, K, mirror,
                                      ws.data_ptr(), ws.numel(), _st()), 'vc_conv_dgrad_f32')
    return din


def _conv_wgrad(prec, det, x, dout, nbr, n_out, ci, co, K):
    L, lib = _lib()
    dw = torch.full((co, K, ci), 7.0, device=DEV)
    if prec == 'bf16':
        if det:
            ws = _ws(lib.vc_conv_wgrad_tc_det_ws_bytes(n_out, ci, co, K))
            fn, name = lib.vc_conv_wgrad_tc_det, 'vc_conv_wgrad_tc_det'
        else:
            ws = _ws(lib.vc_conv_wgrad_tc_ws_bytes(n_out, ci, co, K))
            fn, name = lib.vc_conv_wgrad_tc, 'vc_conv_wgrad_tc'
        L.check(fn(x.data_ptr(), dout.data_ptr(), nbr.data_ptr(), dw.data_ptr(), n_out, ci, co, K, ws.data_ptr(), ws.numel(),
                   _err().data_ptr(), _st()), name)
    else:                            # (the fp32 weight gradient is deterministic already: a two-pass reduction)
        ws = _ws(lib.vc_conv_wgrad_ws_bytes(n_out, ci, co, K))
        L.check(lib.vc_conv_wgrad_f32(x.data_ptr(), dout.data_ptr(), nbr.data_ptr(), dw.data_ptr(), n_out, ci, co, K, ws.data_ptr(),
                                      ws.numel(), _st()), 'vc_conv_wgrad_f32')
    return dw


@pytest.mark.parametrize('det', [0, 1], ids=['normal', 'det'])
@pytest.mark.parametrize('prec', ['bf16', 'fp32'])
@pytest.mark.parametrize('kind', ['subm3d', 'strided', 'many2one'])
def test_conv_nan_inf_rows(ctas, kind, prec, det):
    """one NaN and one +Inf row in the input and in the output gradient: forward, dgrad (the many-to-one table by scatter and
    by gather2d) and wgrad against float64 on the same operands"""
    ci, co = 16, 32
    t = _table(kind)
    nbr, n_in, n_out, K = t['nbr'], t['n_in'], t['n_out'], t['K']
    dt = torch.bfloat16 if prec == 'bf16' else torch.float32
    w = _weights(ci, co, K, 5)
    wr = w.bfloat16().double() if prec == 'bf16' else w.double()
    x = _poisoned(n_in, ci, 6, (n_in // 5, (3 * n_in) // 4), dt)
    if kind == 'many2one':
        # small integers times a power of two per column: the gather form's bf16 per-pixel sums are exact
        g = torch.Generator(device=DEV).manual_seed(7)
        dout = torch.randint(-3, 4, (n_out, co), device=DEV, generator=g).float()
        dout *= torch.pow(2.0, torch.randint(-3, 4, (co,), device=DEV, generator=g).float())
        dout[n_out // 3] = NAN
        dout[(4 * n_out) // 5] = INF
        dout = dout.to(dt)
    else:
        dout = _poisoned(n_out, co, 7, (n_out // 3, (4 * n_out) // 5), dt)
    where = (kind, prec, det, ctas)
    ref = audit.conv(x, wr, nbr, n_out)
    assert not torch.isfinite(ref).all() and torch.isfinite(ref).any()
    match(_conv_fwd(prec, det, x, w, nbr, n_out, ci, co, K), ref, 1e-4, where + ('fwd',))
    din_ref, dw_ref = audit.conv_grads(x, wr, nbr, n_out, dout)
    forms = ('scatter', '2d') if kind == 'many2one' else ('gather',)
    for form in forms:
        match(_conv_dgrad(prec, form, dout, w, t, ci, co), din_ref, 1e-4, where + ('dgrad', form))
    if prec == 'fp32' and det:
        return
    dw = _conv_wgrad(prec, det, x, dout, nbr, n_out, ci, co, K)
    if prec == 'fp32':
        match(dw, dw_ref, 1e-4, where + ('wgrad',))
        return
    # The tensor-core weight gradient multiplies a whole 128-row dout tile with every offset's gathered input rows, the
    # rows of missing pairs zero-filled: a non-finite dout row meets 0 there and makes dw non-finite at offsets where the
    # reference has no pair for that row.  A non-finite INPUT row is gathered only where a pair exists, so it follows the
    # reference exactly.  Run on operands poisoned in some columns only: x NaN in input channels 0-3 and +Inf in 4-7 of two
    # rows, dout NaN in output channels 0-7 and +Inf in 8-15 of two rows.  Then
    #   output channels >= 16 (reached by the x poison only): finiteness equal element by element, tolerance where finite;
    #   output channels < 16: every non-finite value of the reference is non-finite here too (none is lost).
    g = torch.Generator(device=DEV).manual_seed(10)
    xw = torch.randn(n_in, ci, device=DEV, generator=g)
    xw[n_in // 5, :4] = NAN
    xw[(3 * n_in) // 4, 4:8] = INF
    dw_out = torch.randn(n_out, co, device=DEV, generator=g)
    dw_out[n_out // 3, :8] = NAN
    dw_out[(4 * n_out) // 5, 8:16] = INF
    xw, dw_out = xw.bfloat16(), dw_out.bfloat16()
    dw = _conv_wgrad(prec, det, xw, dw_out, nbr, n_out, ci, co, K)
    dw_ref = audit.conv_grads(xw, wr, nbr, n_out, dw_out, need_din=False)[1]
    assert torch.isfinite(dw_ref[16:]).any() and not torch.isfinite(dw_ref[16:]).all()
    match(dw[16:], dw_ref[16:], 1e-4, where + ('wgrad', 'co >= 16'))
    fin, ref_fin = torch.isfinite(dw[:16]).cpu(), torch.isfinite(dw_ref[:16]).cpu()
    assert not (fin & ~ref_fin).any(), where + ('wgrad: a non-finite value was dropped',)
    if fin.any():
        match(dw[:16].cpu()[fin], dw_ref[:16].cpu()[fin], 1e-4, where + ('wgrad', 'co < 16'))


@pytest.mark.parametrize('prec', ['bf16', 'fp32'])
def test_gather2d_ignores_nan_past_the_row_count(ctas, prec):
    """vc_conv_dgrad_gather2d_* with a device row count: NaN in the output-gradient rows past it changes no bit of din"""
    L, lib = _lib()
    cap, n = N, N - 93
    nbr, rep = _table2d(n)
    nd = torch.tensor([n], dtype=torch.int32, device=DEV)
    ci, co = 16, 32
    w = _weights(ci, co, 9, 8)
    tc = prec == 'bf16'
    dt = torch.bfloat16 if tc else torch.float32
    got = []
    for fill in (0.0, NAN):
        dout = torch.randn(cap, co, device=DEV, generator=torch.Generator(device=DEV).manual_seed(9))
        dout[n:] = fill
        dout = dout.to(dt)
        din = torch.full((cap, ci), 7.0, device=DEV)
        ws = _ws(lib.vc_conv_dgrad_gather2d_ws_bytes(cap, ci, co, 9))
        fn = lib.vc_conv_dgrad_gather2d_tc if tc else lib.vc_conv_dgrad_gather2d_f32
        args = (dout.data_ptr(), w.data_ptr(), nbr.data_ptr(), rep.data_ptr(), din.data_ptr(), cap, nd.data_ptr(), ci, co, 9,
                ws.data_ptr(), ws.numel()) + ((_err().data_ptr(),) if tc else ()) + (_st(),)
        L.check(fn(*args), 'gather2d dgrad')
        torch.cuda.synchronize()
        got.append(din)
    assert torch.isfinite(got[0]).all() and torch.equal(got[0], got[1])


@pytest.mark.parametrize('col', [0, 16])
def test_conv_ignores_nan_beside_a_column_slice(ctas, col):
    """The tensor-core conv forward and deterministic wgrad read their input as a column slice of a wider matrix (row pitch
    in_ld > cin, as the plan executor reads an in-place concat): NaN in the other columns against zeros there changes no
    bit, and the result equals the conv of the dense slice"""
    L, lib = _lib()
    ci, co, ld = 16, 32, 48
    t = _table('subm3d')
    nbr, n, K = t['nbr'], t['n_in'], t['K']
    w = _weights(ci, co, K, 30)
    g = torch.Generator(device=DEV).manual_seed(31)
    body = torch.randn(n, ci, device=DEV, generator=g).bfloat16()
    dout = torch.randn(n, co, device=DEV, generator=g).bfloat16()
    runs = []
    for fill in (0.0, NAN):
        wide = torch.full((n, ld), fill, device=DEV).bfloat16()
        wide[:, col:col + ci] = body
        xs = wide[:, col:]
        out = torch.full((n, co), 7.0, device=DEV)
        ws = _ws(lib.vc_conv_tc_ws_bytes(ci, co, K))
        L.check(lib.vc_conv_fwd_tc_ld(xs.data_ptr(), ld, w.data_ptr(), nbr.data_ptr(), out.data_ptr(), n, ci, co, K, None, ws.data_ptr(),
                                      ws.numel(), _err().data_ptr(), _st()), 'vc_conv_fwd_tc_ld')
        dw = torch.full((co, K, ci), 7.0, device=DEV)
        ws = _ws(lib.vc_conv_wgrad_tc_det_ws_bytes(n, ci, co, K))
        L.check(lib.vc_conv_wgrad_tc_det_ld(xs.data_ptr(), ld, dout.data_ptr(), nbr.data_ptr(), dw.data_ptr(), n, ci, co, K,
                                            ws.data_ptr(), ws.numel(), _err().data_ptr(), _st()), 'vc_conv_wgrad_tc_det_ld')
        torch.cuda.synchronize()
        runs.append((out, dw))
    (o0, w0), (o1, w1) = runs
    assert torch.isfinite(o0).all() and torch.isfinite(w0).all()
    assert torch.equal(o0, o1) and torch.equal(w0, w1)
    assert torch.equal(o0, _conv_fwd('bf16', 0, body, w, nbr, n, ci, co, K))
    assert torch.equal(w0, _conv_wgrad('bf16', 1, body, dout, nbr, n, ci, co, K))


# ------------------------------------------------------------------------------------------------ BatchNorm + ReLU
EPS, MOM = 1e-3, 0.01


def _bn_params(c, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (0.5 + torch.rand(c, device=DEV, generator=g), 0.1 * torch.randn(c, device=DEV, generator=g),
            0.1 * torch.randn(c, device=DEV, generator=g), 0.5 + torch.rand(c, device=DEV, generator=g))


def _bn_ref(x, gamma, beta, rm0, rv0, training):
    """torch BatchNorm1d + ReLU in float64 -> (y, stats [4, c] = scale, shift, mean, invstd, running_mean, running_var)"""
    x = x.double()
    rm, rv = rm0.double().clone(), rv0.double().clone()
    y = torch.relu(F.batch_norm(x, rm, rv, gamma.double(), beta.double(), bool(training), MOM, EPS))
    if training:
        mean, invstd, _, _ = audit.batch_stats(x, EPS)
    else:
        mean, invstd = rm0.double(), 1.0 / torch.sqrt(rv0.double() + EPS)
    scale = gamma.double() * invstd
    return y, torch.stack([scale, beta.double() - mean * scale, mean, invstd]), rm, rv


def _bn_x(n, c, seed):
    """randn with a NaN in channel 1, +Inf in channel 2 and -Inf in channel 3 (one row each)"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(n, c, device=DEV, generator=g)
    x[n // 3, 1] = NAN
    x[n // 2, 2] = INF
    x[(2 * n) // 3, 3] = -INF
    return x


def _check_bn_outputs(got, x, gamma, beta, rm0, rv0, training, where):
    y_ref, st_ref, rm_ref, rv_ref = _bn_ref(x, gamma, beta, rm0, rv0, training)
    match(got['y'], y_ref, 1e-5, where + ('y',))
    match(got['yb'].float(), y_ref, 2.0 ** -8, where + ('yb',))
    fin = torch.isfinite(got['y'])
    assert torch.equal(got['yb'][fin], got['y'][fin].bfloat16()), where
    match(got['stats'], st_ref, 1e-5, where + ('stats',))
    match(got['rm'], rm_ref, 1e-6, where + ('running_mean',))
    match(got['rv'], rv_ref, 1e-6, where + ('running_var',))


@pytest.mark.parametrize('training', [1, 0], ids=['train', 'eval'])
def test_bn_apply_relu(training):
    """vc_bn_apply_relu_f32: NaN / +Inf / -Inf in three channels; y, yb, the stats block and the running buffers"""
    L, lib = _lib()
    n, c = N, 32
    x = _bn_x(n, c, 11)
    gamma, beta, rm0, rv0 = _bn_params(c, 12)
    rm, rv = rm0.clone(), rv0.clone()
    xd = x.double()
    sums = torch.stack([xd.sum(0), (xd * xd).sum(0)]).contiguous()           # what the conv's epilogue accumulates
    y = torch.full((n, c), 7.0, device=DEV)
    yb = torch.full((n, c), 7.0, dtype=torch.bfloat16, device=DEV)
    stats = torch.empty(4, c, device=DEV)
    nbt = torch.zeros(1, dtype=torch.int64, device=DEV)
    L.check(lib.vc_bn_apply_relu_f32(x.data_ptr(), sums.data_ptr(), n, c, gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr(),
                                     nbt.data_ptr(), MOM, EPS, training, y.data_ptr(), yb.data_ptr(), stats.data_ptr(), 1, _st()),
            'vc_bn_apply_relu_f32')
    torch.cuda.synchronize()
    _check_bn_outputs(dict(y=y, yb=yb, stats=stats, rm=rm, rv=rv), x, gamma, beta, rm0, rv0, training, ('apply', training))
    if not training:
        assert torch.isnan(y[n // 3, 1]) and y[n // 2, 2] == INF and y[(2 * n) // 3, 3] == 0


def _conv_bn_relu(lib, L, xb, w, nbr, cap, n_dev, ci, co, det, training, params):
    from virconv_b200 import ops
    gamma, beta, rm0, rv0 = params
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.zeros(1, dtype=torch.int64, device=DEV)
    x = torch.full((cap, co), 7.0, device=DEV)
    y = torch.full((cap, co), 7.0, device=DEV)
    yb = torch.full((cap, co), 7.0, dtype=torch.bfloat16, device=DEV)
    stats = torch.empty(4, co, device=DEV)
    nd = torch.tensor([n_dev], dtype=torch.int32, device=DEV) if n_dev is not None else None
    ws = _ws(lib.vc_conv_bn_relu_tc_ws_bytes(cap, ci, co, 27))
    L.check(lib.vc_conv_bn_relu_tc(xb.data_ptr(), w.data_ptr(), nbr.data_ptr(), x.data_ptr(), cap, ops._p(nd), ci, co, 27, det,
                                   gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr(), nbt.data_ptr(), MOM, EPS, training,
                                   y.data_ptr(), co, yb.data_ptr(), co, stats.data_ptr(), ws.data_ptr(), ws.numel(), _err().data_ptr(),
                                   ops._stream()), 'vc_conv_bn_relu_tc')
    torch.cuda.synchronize()
    return dict(x=x, y=y, yb=yb, stats=stats, rm=rm, rv=rv, nbt=nbt)


@pytest.fixture
def bn_fused_flag():
    L, lib = _lib()
    yield lambda f: lib.vc_set_conv_bn_fused(f)
    import os
    lib.vc_set_conv_bn_fused(int(os.environ.get('VIRCONV_CONV_BN_FUSED', '1') != '0'))


@pytest.mark.parametrize('training', [1, 0], ids=['train', 'eval'])
@pytest.mark.parametrize('det', [0, 1])
@pytest.mark.parametrize('fused', [1, 0], ids=['fused', 'unfused'])
def test_conv_bn_relu_tc(ctas, bn_fused_flag, fused, det, training):
    """vc_conv_bn_relu_tc with a NaN, a +Inf and a -Inf input row: x against the float64 conv, then y, yb, stats and the
    running buffers against torch's BatchNorm1d + ReLU of that x"""
    L, lib = _lib()
    bn_fused_flag(fused)
    ci, co = 16, 32
    nbr = _table('subm3d')['nbr']
    w = _weights(ci, co, 27, 13)
    g = torch.Generator(device=DEV).manual_seed(14)
    xb = torch.randn(N, ci, device=DEV, generator=g)
    xb[N // 4] = NAN
    xb[N // 2, :8] = INF
    xb[(3 * N) // 4, 8:] = -INF
    xb = xb.bfloat16()
    params = _bn_params(co, 15)
    got = _conv_bn_relu(lib, L, xb, w, nbr, N, None, ci, co, det, training, params)
    where = ('conv_bn_relu', fused, det, training, ctas)
    x_ref = audit.conv(xb, w.bfloat16().double(), nbr, N)
    match(got['x'], x_ref, 1e-4, where + ('x',))
    assert torch.isfinite(got['x']).any() and not torch.isfinite(got['x']).all()
    # BN of the kernel's own x (its finite rows are within 1e-4 of the float64 conv)
    _check_bn_outputs(got, got['x'], *params, training, where)
    assert int(got['nbt'].item()) == training


@pytest.mark.parametrize('training', [1, 0], ids=['train', 'eval'])
def test_conv_bn_relu_ignores_nan_past_the_row_count(ctas, bn_fused_flag, training):
    """NaN input rows past the device row count (the table's tail is -1) against zeros there: every output bit for bit"""
    L, lib = _lib()
    bn_fused_flag(1)
    ci, co = 16, 32
    cap, n = N, N - 77
    nbr = torch.full((27, cap), -1, dtype=torch.int32, device=DEV)
    from virconv_b200 import ops
    nbr[:, :n] = ops.build_subm_rulebook(_coords3(N, 21)[:n].contiguous(), 2, SHAPE3, 3).nbr
    w = _weights(ci, co, 27, 16)
    params = _bn_params(co, 17)
    runs = []
    for fill in (0.0, NAN):
        g = torch.Generator(device=DEV).manual_seed(18)
        xb = torch.randn(cap, ci, device=DEV, generator=g)
        xb[n:] = fill
        runs.append(_conv_bn_relu(lib, L, xb.bfloat16(), w, nbr, cap, n, ci, co, 1, training, params))
    a, b = runs
    for k in a:
        if k == 'x':
            assert torch.equal(a[k][:n], b[k][:n]), k
        else:
            assert torch.isfinite(a[k]).all() and torch.equal(a[k], b[k]), k


@pytest.mark.parametrize('training', [1, 0], ids=['train', 'eval'])
@pytest.mark.parametrize('det', [0, 1])
@pytest.mark.parametrize('fused', [1, 0], ids=['fused', 'unfused'])
def test_bn_relu_bwd(fused, det, training):
    """vc_bn_relu_bwd_f32 / vc_bn_relu_bwd_det_f32 (dx, dgamma, dbeta) against autograd through torch's BatchNorm1d + ReLU
    in float64: x with NaN / +Inf / -Inf in three channels, a NaN in one gradient row"""
    L, lib = _lib()
    L.check(lib.vc_set_bn_fused(fused), 'vc_set_bn_fused')
    try:
        n, c = N, 32
        x = _bn_x(n, c, 21)
        gamma, beta, rm0, rv0 = _bn_params(c, 22)
        g = torch.Generator(device=DEV).manual_seed(23)
        dy = torch.randn(n, c, device=DEV, generator=g)
        dy[n // 5, 0] = NAN
        # the forward's stats block, from the float64 reference (what the kernel reads: scale, shift, mean, invstd)
        _, st, _, _ = _bn_ref(x, gamma, beta, rm0, rv0, training)
        stats = st.float().contiguous()
        dx = torch.full((n, c), 7.0, device=DEV)
        dxb = torch.full((n, c), 7.0, dtype=torch.bfloat16, device=DEV)
        dgamma = torch.full((c,), 7.0, device=DEV)
        dbeta = torch.full((c,), 7.0, device=DEV)
        if det:
            ws = _ws(lib.vc_bn_bwd_det_ws_bytes(n, c))
            L.check(lib.vc_bn_relu_bwd_det_f32(dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), stats.data_ptr(), dx.data_ptr(),
                                               dxb.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), n, c, training, ws.data_ptr(),
                                               ws.numel(), _st()), 'vc_bn_relu_bwd_det_f32')
        else:
            bsums = torch.zeros(2, c, dtype=torch.float64, device=DEV)
            L.check(lib.vc_bn_relu_bwd_f32(dy.data_ptr(), x.data_ptr(), None, gamma.data_ptr(), stats.data_ptr(), dx.data_ptr(),
                                           dxb.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), n, c, training, bsums.data_ptr(),
                                           _st()), 'vc_bn_relu_bwd_f32')
        torch.cuda.synchronize()
    finally:
        lib.vc_set_bn_fused(1)
    # the reference: autograd, with the saved statistics (the kernel's stats block) held as the forward had them
    xd = x.double().requires_grad_(True)
    gd = gamma.double().requires_grad_(True)
    bd = beta.double().requires_grad_(True)
    if training:
        y = torch.relu(F.batch_norm(xd, None, None, gd, bd, True, 0.0, EPS))
    else:
        y = torch.relu(F.batch_norm(xd, rm0.double(), rv0.double(), gd, bd, False, 0.0, EPS))
    y.backward(dy.double())
    where = ('bn_bwd', fused, det, training)
    match(dx, xd.grad, 1e-5, where + ('dx',))
    match(dxb.float(), xd.grad, 2.0 ** -8, where + ('dx_bf16',))
    match(dgamma, gd.grad, 1e-5, where + ('dgamma',))
    match(dbeta, bd.grad, 1e-5, where + ('dbeta',))


# ------------------------------------------------------------------------------------------------ voxel-RoI pooling
@pytest.fixture
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.mark.parametrize('det', [False, True], ids=['atomic', 'det'])
def test_voxel_pool_nan_feature_row(no_tf32, det):
    """the fused pooling with one NaN feature row: pooled is NaN exactly where max_pool2d over the float64 grouping is, and
    the backward (differentiated at the kernel's argmax) sends the gradient of those maxima to the NaN row"""
    from oracle import voxel_pool as o
    from test_gpu_roi_pool import _scene
    from virconv_b200 import voxel_pool
    xyz, xyz_cnt, new_xyz, new_cnt, new_coords, v2p = (torch.from_numpy(a).cuda() for a in _scene(3))
    N_, C, ns, max_range, radius = xyz.shape[0], 32, 16, (2, 2, 2), 0.4
    torch.manual_seed(0)
    mlp_pos = torch.nn.Sequential(torch.nn.Conv2d(3, C, 1, bias=False), torch.nn.BatchNorm2d(C)).cuda().train()
    with torch.no_grad():
        mlp_pos[1].weight.uniform_(0.5, 1.5)
        mlp_pos[1].bias.uniform_(-0.3, 0.3)
    p0 = {k: v.detach().double().clone() for k, v in mlp_pos.state_dict().items()}
    feats = torch.randn(N_, C, device='cuda')
    idx, empty, _ = voxel_pool.voxel_pool_query(max_range, radius, ns, xyz, new_xyz, new_coords, v2p, False)
    hits = torch.bincount(idx[~empty.bool()].reshape(-1).long(), minlength=N_)
    bad = int(hits.argmax())                             # the row in the most balls
    feats[bad] = NAN
    feats.requires_grad_(True)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        pooled, argmax, idx, empty, mom = voxel_pool.voxel_pool(feats, xyz, new_xyz, new_coords, v2p, mlp_pos, max_range, radius, ns)
        go = torch.randn(pooled.shape[0], C, device='cuda')
        pooled.backward(go)
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)

    def params64():
        p = {'mlps_pos.0.' + k: v.clone() for k, v in p0.items()}
        for k in ('0.weight', '1.weight', '1.bias'):
            p['mlps_pos.0.' + k].requires_grad_(True)
        return p
    keep = {}
    with torch.no_grad():
        o.pool(params64(), 0, max_range, radius, ns, feats.detach().double(), xyz.double(), xyz_cnt, new_xyz.double(), new_cnt,
               new_coords, v2p, True, query=(idx, empty), keep=keep)
    ref = keep['pooled'][0]
    assert torch.isnan(ref).any() and torch.isfinite(ref).any()
    match(pooled, ref, 1e-5, ('pooled', det))
    v = keep['v'][0]
    at = v.gather(2, argmax.long().unsqueeze(-1)).squeeze(-1)
    assert torch.equal(torch.isnan(at), torch.isnan(ref))            # the argmax of a NaN maximum is a NaN slot
    p64 = params64()
    f64 = feats.detach().double().requires_grad_(True)
    r = o.pool(p64, 0, max_range, radius, ns, f64, xyz.double(), xyz_cnt, new_xyz.double(), new_cnt, new_coords, v2p, True,
               query=(idx, empty), argmax=argmax)
    r.squeeze(0).t().backward(go.double())
    match(feats.grad, f64.grad, 1e-4, ('grad_features', det))
    assert feats.grad[bad].abs().sum() > 0
    for name, prm in (('0.weight', mlp_pos[0].weight), ('1.weight', mlp_pos[1].weight), ('1.bias', mlp_pos[1].bias)):
        match(prm.grad, p64['mlps_pos.0.' + name].grad, 1e-4, (name, det))


# ------------------------------------------------------------------------------------------------ masked_mean
def test_masked_mean_nan_inside_and_past_the_count():
    from virconv_b200.graph import _MaskedMean
    cap, c, n = 1000, 16, 777
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(cap, c, generator=g) * 3 + 0.5).cuda()
    x[n:] = NAN
    nd = torch.tensor([n], dtype=torch.int32, device=DEV)
    m = _MaskedMean.apply(x, nd)
    want = x[:n].double().mean().item()
    assert np.isfinite(m.item()) and abs(m.item() - want) <= 1e-6 * abs(want)
    x[n - 1, 3] = NAN
    assert np.isnan(_MaskedMean.apply(x, nd).item())
    x[n - 1, 3] = INF
    assert not np.isfinite(_MaskedMean.apply(x, nd).item())


# ------------------------------------------------------------------------------------------------ voxeliser
RANGE = (0, -40, -3, 70.4, 40, 1)


def _voxeliser_points():
    """two samples of a scene, with points that carry NaN / +-Inf in x, y and z, NaN in a feature column (the last one,
    which the max-VFE reads, and one before it), and points exactly on the lower and upper bounds and one float32 ulp
    below the upper bound"""
    from virconv_b200 import scenes
    per = []
    for b, sid in enumerate([3, 4]):
        p = scenes.make_points(sid, 2048, 3000).astype(np.float32)
        k = 0
        for d in range(3):
            for v in (NAN, INF, -INF):
                p[10 + k, d] = v
                k += 1
        p[40, :3] = (10.0, 0.0, -1.0)
        p[40, p.shape[1] - 1] = NAN
        p[41, :3] = (12.0, 0.0, -1.0)
        p[41, 3] = NAN
        p[42, :3] = RANGE[:3]
        p[43, :3] = (RANGE[3], 10.0, -1.0)
        p[44, :3] = (20.0, RANGE[4], -1.0)
        p[45, :3] = (np.nextafter(np.float32(RANGE[3]), np.float32(0)), 10.0, -1.0)
        p[46, :3] = (20.0, np.nextafter(np.float32(RANGE[4]), np.float32(0)), -1.0)
        p[47, :3] = (30.0, 0.0, np.nextafter(np.float32(RANGE[5]), np.float32(0)))
        per.append(p)
    return per


def _voxeliser_reference(per, model):
    from virconv_b200 import scenes
    want = []
    with np.errstate(invalid='ignore'):
        for b, p in enumerate(per):
            vox, coords, num = scenes.voxelize_first_come(scenes.mask_points_by_range(p, RANGE), pc_range=RANGE)
            want.append((scenes.mean_vfe(vox, num, model), np.concatenate([np.full((len(coords), 1), b, np.int32), coords], 1), num))
    return [np.concatenate([w[i] for w in want]) for i in range(3)]


def _same_nan(a, b):
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize('model', ['max', None])
def test_voxelize_mean_nonfinite_points(model):
    from virconv_b200 import ops
    per = _voxeliser_points()
    wf, wc, wn = _voxeliser_reference(per, model)
    assert np.isnan(wf).any()                                   # the NaN-feature points are kept
    pts = torch.from_numpy(np.concatenate([np.concatenate([np.full((len(p), 1), b, np.float32), p], 1)
                                           for b, p in enumerate(per)])).to(DEV)
    f, c, nm = ops.voxelize_mean(pts, 2, RANGE, vfe_model=model)
    assert np.array_equal(c.cpu().numpy(), wc)
    assert np.array_equal(nm.cpu().numpy(), wn)
    assert _same_nan(f.cpu().numpy(), wf)


def test_voxelize_mean_captured_nonfinite_points():
    """the static form GraphedStep(voxelizer=...) runs inside its graph: captured once, replayed on the points above in a
    capacity-sized buffer with an out-of-range tail"""
    from virconv_b200 import ops
    per = _voxeliser_points()
    wf, wc, wn = _voxeliser_reference(per, 'max')
    pts = np.concatenate([np.concatenate([np.full((len(p), 1), b, np.float32), p], 1) for b, p in enumerate(per)])
    cap = len(pts) + 500
    buf = torch.zeros(cap, pts.shape[1], device=DEV)
    buf[:, 0] = 1
    buf[:, 1:4] = -1.0e6
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.voxelize_mean(buf, 2, RANGE, max_voxels=8000, vfe_model='max', static=True)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        f, c, nm, n_out = ops.voxelize_mean(buf, 2, RANGE, max_voxels=8000, vfe_model='max', static=True)
    buf[:len(pts)] = torch.from_numpy(pts).to(DEV)
    graph.replay()
    torch.cuda.synchronize()
    m = int(n_out.item())
    assert m == len(wn)
    assert np.array_equal(c[:m].cpu().numpy(), wc) and np.array_equal(nm[:m].cpu().numpy(), wn)
    assert _same_nan(f[:m].cpu().numpy(), wf)
    assert bool((f[m:] == 0).all()) and bool((c[m:] == -1).all())


# ------------------------------------------------------------------------------------------------ whole training steps
def _model(which):
    from virconv_b200.backbone import VirConv8x, VirConvL8x
    if which == 'L':
        m = VirConvL8x(CFG_L, 8, [1408, 1600, 80], precision='bf16')
        fill_module(m, 666)
    else:
        m = VirConv8x(CFG_T, 8, [1408, 1600, 80], precision='bf16', discard_mode='paper', discard_rng='device')
        fill_module(m, 667)
    return m.to(DEV).train()


def _batch(which, ids):
    from virconv_b200 import scenes
    if which == 'L':
        b = scenes.make_batch(ids, n_lidar=4096, n_virtual=9000, max_voxels=7000, training=True)
        return {'voxel_features': torch.from_numpy(b.voxel_features.copy()).to(DEV),
                'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).to(DEV), 'batch_size': b.batch_size, 'calib': b.calib,
                'aug_param': torch.from_numpy(b.aug_param.copy())}
    b = scenes.make_batch_mm(ids, max_voxels=3000, training=True, n_lidar=4096, n_virtual=6000)
    bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
    bd.update(batch_size=b.batch_size, calib=b.calib, aug_param=torch.from_numpy(b.aug_param.copy()),
              stvd_seed=torch.tensor([1234], dtype=torch.int64, device=DEV))
    return bd


def _loss(out):
    from virconv_b200.graph import masked_mean
    ts = [out['encoded_spconv_tensor']]
    for g in ('multi_scale_3d_features', 'multi_scale_3d_features_mm'):
        ts += list(out.get(g, {}).values())
    return sum(masked_mean(t) for t in ts)


class _Eager:
    """the plan executor without a graph, then the fused update's eager step()"""

    def __init__(self, model, opt):
        self.model, self.opt = model, opt

    def __call__(self, batch):
        self.opt.zero_grad()
        loss = _loss(self.model(dict(batch)))
        loss.backward()
        self.opt.step(max_norm=10.0)
        return loss.detach()


@pytest.mark.parametrize('bad', [NAN, INF], ids=['nan', 'inf'])
@pytest.mark.parametrize('mode', ['eager', 'graphed'])
@pytest.mark.parametrize('which', ['L', 'T'])
def test_poisoned_batch_is_skipped(which, mode, bad):
    """batches clean, poisoned (one voxel feature NaN or +Inf), clean: the poisoned step reports a non-finite loss and norm,
    is counted as skipped and leaves parameters and Adam moments bit-identical; its forward still ran, so BatchNorm running
    buffers hold non-finite values, as torch leaves them.  The next clean step equals that of a twin that never saw the
    poisoned batch."""
    from virconv_b200.graph import GraphedStep
    from virconv_b200.optim import FusedAdamOneCycle
    clean = [_batch(which, [1, 2]), _batch(which, [3, 4])]
    poisoned = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in clean[1].items()}
    poisoned['voxel_features'][17, 1] = bad
    torch.use_deterministic_algorithms(True)
    try:
        models = [_model(which), _model(which)]
        opts = [FusedAdamOneCycle.from_model(m, wd=0.01) for m in models]
        if mode == 'eager':
            steps = [_Eager(m, o) for m, o in zip(models, opts)]
        else:
            steps = [GraphedStep(m, _loss, margin=1.35, grain=256, optimizer=o, max_grad_norm=10.0) for m, o in zip(models, opts)]
        for s in steps:
            s(clean[0])
        torch.cuda.synchronize()
        assert opts[0].applied_steps() == 1 == opts[1].applied_steps()
        before = [p.detach().clone() for p in models[0].parameters()] + [opts[0].exp_avg_flat.clone(), opts[0].exp_avg_sq_flat.clone()]
        bufs_before = {k: b.clone() for k, b in models[0].named_buffers() if b.is_floating_point()}
        loss = float(steps[0](poisoned))
        torch.cuda.synchronize()
        assert not np.isfinite(loss) and not np.isfinite(float(opts[0].last_total_norm))
        assert opts[0].skipped_steps() == 1 and opts[0].applied_steps() == 1
        after = [p.detach() for p in models[0].parameters()] + [opts[0].exp_avg_flat, opts[0].exp_avg_sq_flat]
        assert all(torch.equal(a, b) for a, b in zip(before, after))
        changed = [k for k, b in models[0].named_buffers() if k in bufs_before and not torch.isfinite(b).all()]
        assert changed, 'the poisoned forward should leave non-finite BatchNorm running statistics'
        assert all(torch.isfinite(b).all() for b in bufs_before.values())
        losses = [float(s(clean[1])) for s in steps]
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    assert np.isfinite(losses[0]) and losses[0] == losses[1]
    assert opts[0].applied_steps() == 2 == opts[1].applied_steps() and opts[1].skipped_steps() == 0
    assert float(opts[0].last_total_norm) == float(opts[1].last_total_norm)
    bad_p = [k for (k, p), q in zip(models[0].named_parameters(), models[1].parameters()) if not torch.equal(p, q)]
    assert not bad_p, bad_p[:5]
    assert torch.equal(opts[0].exp_avg_flat, opts[1].exp_avg_flat) and torch.equal(opts[0].exp_avg_sq_flat, opts[1].exp_avg_sq_flat)


def _oracle_named(which, o):
    if which == 'L':
        named = {'out': o['out']}
        named.update({'multi_scale_3d_features:x_conv%d' % i: o['x_conv%d' % i] for i in range(1, 5)})
        return named
    named = {'out': o['encoded_spconv_tensor']}
    for g in ('multi_scale_3d_features', 'multi_scale_3d_features_mm'):
        for k, t in o.get(g, {}).items():
            if t is not None:
                named[f'{g}:{k}'] = t
    return named


@pytest.mark.parametrize('which', ['L', 'T'])
def test_graphed_forward_eval_publishes_nan(which):
    """GraphedForward(model.eval()) on a batch with one NaN voxel feature: every published tensor is non-finite exactly where
    the float64 module path (oracle.backbone on the CPU, the same weights and running statistics) is, matched by
    coordinates"""
    from oracle import backbone as ob
    from oracle.testing import join_by_coords
    from virconv_b200 import scenes
    from virconv_b200.graph import GraphedForward
    if which == 'L':
        m = _model('L').eval()
        b = scenes.make_batch([3, 4], n_lidar=4096, n_virtual=6000, max_voxels=3000, training=False)
        arrays = {'voxel_features': b.voxel_features.copy(), 'voxel_coords': b.voxel_coords.copy()}
        ref_m = ob.VirConvL8x()
    else:
        from virconv_b200.backbone import VirConv8x
        m = VirConv8x(CFG_T, 8, [1408, 1600, 80], precision='bf16')
        fill_module(m, 667)
        m = m.to(DEV).eval()
        b = scenes.make_batch_mm([3, 4], max_voxels=3000, training=False, rot_num=1, n_lidar=4096, n_virtual=6000)
        arrays = {k: v.copy() for k, v in b.arrays.items()}
        ref_m = ob.VirConv8x()
    arrays['voxel_features'][17, 1] = np.nan
    if which == 'T':
        arrays['voxel_features_mm'][23, 2] = np.nan
    batch = {k: torch.from_numpy(v).to(DEV) for k, v in arrays.items()}
    batch.update(batch_size=b.batch_size, calib=b.calib)
    if which == 'T':
        batch['transform_param'] = torch.from_numpy(b.transform_param.copy()).to(DEV)
    out = GraphedForward(m, margin=1.3, grain=256)(batch)
    torch.cuda.synchronize()
    ref_m.load_state_dict({k: v.cpu() for k, v in m.state_dict().items()})
    ref_m = ref_m.double().eval()
    cpu = {k: torch.from_numpy(v) for k, v in arrays.items()}
    with torch.no_grad():
        if which == 'L':
            o = ref_m(cpu['voxel_features'].double(), cpu['voxel_coords'], b.batch_size, b.calib)
        else:
            cpu = {k: (v.double() if v.is_floating_point() and 'features' in k else v) for k, v in cpu.items()}
            o = ref_m(cpu, b.batch_size, b.calib, transform_param=torch.from_numpy(b.transform_param.copy()))
    ref = _oracle_named(which, o)
    got = {'out': out['encoded_spconv_tensor']}
    for g in ('multi_scale_3d_features', 'multi_scale_3d_features_mm'):
        for k, t in out.get(g, {}).items():
            if t is not None:
                got[f'{g}:{k}'] = t
    assert sorted(got) == sorted(ref)
    nonfinite = 0
    for k, r in ref.items():
        t = got[k]
        rows = int(t.num_rows.item())
        gf, rf = join_by_coords(t.indices[:rows].cpu().numpy(), t.features[:rows].detach().cpu(), r.indices.numpy(), r.features)
        fin_ref = torch.isfinite(rf)
        assert torch.equal(torch.isfinite(gf), fin_ref), (k, int((torch.isfinite(gf) != fin_ref).sum()))
        nonfinite += int((~fin_ref).sum())
        assert fin_ref.any(), k
    assert nonfinite > 0
