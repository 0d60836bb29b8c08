"""The persistent tensor-core conv kernels through the C ABI at ~330 000 rows (2 578+ tiles of 128 rows): every CTA runs
many tiles (>= 9 at two CTAs per SM, >= 19 at one), so the neighbour-table ring wraps, the mbarrier phases cycle across
tiles and each CTA's BatchNorm partials cover several tiles.  Each result is compared with the float64 reference fed the
same bf16 operands (oracle.audit: spconv_cpu.native_conv and its autograd gradients), rel_err < 1e-4.

Shapes: row counts = 1, 2, 3 mod 4 (the scalar neighbour-table loads) and 1, 127 mod 128 (a last, nearly empty or nearly
full tile); a band of isolated voxels that fills whole tiles with the centre offset only; the backbone's channel pairs."""
import time

import numpy as np
import pytest
import torch

from oracle import audit
from oracle.testing import rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
N0 = 128 * 2578                      # 329 984 rows
COUNTS = (N0 + 1, N0 + 2, N0 + 127, N0 + 3)     # = 1, 2, 3 mod 4 and 1, 127 mod 128
BAND_AT, BAND = 1250 * 128, 1000     # isolated voxels: rows [BAND_AT, BAND_AT + BAND), whole tiles 1250-1256
SHAPE3 = [24, 192, 192]
SHAPE2 = [200, 704]
PAIRS = ((8, 8), (8, 16), (16, 16), (16, 32), (32, 32), (32, 64), (64, 64))
TOL = dict(out=1e-4, mean=1e-5, invstd=1e-5, y=1e-5, running=1e-6)
WORST = {}


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


def _note(name, value, limit, where):
    WORST[name] = max(WORST.get(name, 0.0), float(value))
    assert value < limit, (name, where, float(value), limit)


@pytest.fixture(scope='module', autouse=True)
def _report():
    t0 = time.time()
    yield
    print('\n[tc multitile] %.1f s: ' % (time.time() - t0) + ', '.join('%s %.3g' % kv for kv in sorted(WORST.items())))


@pytest.fixture(params=[1, 2], ids=['1cta', '2cta'])
def ctas(request):
    L, lib = _lib()
    L.check(lib.vc_conv_tc2_config(request.param), 'vc_conv_tc2_config')
    try:
        yield request.param
    finally:
        lib.vc_conv_tc2_config(0)
    assert int(_err().item()) == 0


@pytest.fixture(scope='module')
def coords3():
    """[COUNTS[-2], 4] int32 (b, z, y, x): two scenes at ~20 % occupancy (x < 160), with BAND isolated voxels (every
    coordinate a multiple of 3, x >= 165: no neighbour within one voxel) at rows BAND_AT..BAND_AT + BAND"""
    rng = np.random.default_rng(11)
    need = max(COUNTS) - BAND
    cells = rng.choice(2 * SHAPE3[0] * SHAPE3[1] * 160, size=need, replace=False)
    b, r = np.divmod(cells, SHAPE3[0] * SHAPE3[1] * 160)
    z, r = np.divmod(r, SHAPE3[1] * 160)
    y, x = np.divmod(r, 160)
    main = np.stack([b, z, y, x], 1)
    g = np.stack(np.meshgrid(np.arange(0, SHAPE3[0], 3), np.arange(0, SHAPE3[1], 3), np.arange(165, SHAPE3[2], 3),
                             indexing='ij'), -1).reshape(-1, 3)
    band = np.concatenate([np.zeros((BAND, 1), np.int64), g[rng.choice(g.shape[0], BAND, replace=False)]], 1)
    co = np.concatenate([main[:BAND_AT], band, main[BAND_AT:]]).astype(np.int32)
    return torch.from_numpy(co).to(DEV)


def _subm(coords, n):
    from virconv_b200 import ops
    return ops.build_subm_rulebook(coords[:n].contiguous(), 2, SHAPE3, 3).nbr


def _weights(ci, co, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(co, K, ci, device=DEV, generator=g) * (2.0 / (K * ci)) ** 0.5).contiguous()


def _feats(n, c, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(n, c, device=DEV, generator=g).bfloat16()


def test_centre_band_fills_whole_tiles(coords3):
    nbr = _subm(coords3, COUNTS[0])
    rows = nbr[:, BAND_AT:BAND_AT + BAND]
    assert bool((rows[13] == torch.arange(BAND_AT, BAND_AT + BAND, device=DEV, dtype=torch.int32)).all())
    assert bool((rows[torch.arange(27) != 13] == -1).all())
    assert (BAND // 128) >= 7 and BAND_AT % 128 == 0


@pytest.mark.parametrize('p', range(len(PAIRS)), ids=['%dx%d' % pc for pc in PAIRS])
def test_fwd_and_mirrored_dgrad(coords3, ctas, p):
    """vc_conv_fwd_tc and vc_conv_dgrad_tc (mirror=1 on the submanifold table itself), one row count per pair"""
    L, lib = _lib()
    ci, co = PAIRS[p]
    n = COUNTS[p % len(COUNTS)]
    nbr = _subm(coords3, n)
    w = _weights(ci, co, 27, p)
    wb = w.bfloat16().double()
    xb = _feats(n, ci, 100 + p)
    out = torch.full((n, co), float('nan'), device=DEV)
    ws = _ws(lib.vc_conv_tc_ws_bytes(ci, co, 27))
    L.check(lib.vc_conv_fwd_tc(xb.data_ptr(), w.data_ptr(), nbr.data_ptr(), out.data_ptr(), n, ci, co, 27, None, ws.data_ptr(),
                               ws.numel(), _err().data_ptr(), _st()), 'vc_conv_fwd_tc')
    _note('fwd', rel_err(out, audit.conv(xb, wb, nbr, n)) / TOL['out'], 1, (ci, co, n))
    dob = _feats(n, co, 200 + p)
    din = torch.full((n, ci), float('nan'), device=DEV)
    L.check(lib.vc_conv_dgrad_tc(dob.data_ptr(), w.data_ptr(), nbr.data_ptr(), din.data_ptr(), n, ci, co, 27, 1, ws.data_ptr(),
                                 ws.numel(), _err().data_ptr(), _st()), 'vc_conv_dgrad_tc')
    ref = audit.conv_grads(torch.zeros(n, ci, device=DEV), wb, nbr, n, dob)[0]
    _note('dgrad_mirror', rel_err(din, ref) / TOL['out'], 1, (ci, co, n))


@pytest.mark.parametrize('ci,co', [(16, 32), (32, 64), (64, 64)])
def test_strided_dgrad(coords3, ctas, ci, co):
    """vc_conv_dgrad_tc over a stride-2 conv's nbr_bwd table (the offset-scanning path)"""
    from virconv_b200 import ops
    L, lib = _lib()
    n = COUNTS[3]
    rb = ops.build_conv_rulebook(coords3[:n].contiguous(), 2, SHAPE3, 3, 2, 1)
    w = _weights(ci, co, 27, ci + co)
    dob = _feats(rb.n_out, co, 300 + ci)
    din = torch.full((n, ci), float('nan'), device=DEV)
    ws = _ws(lib.vc_conv_tc_ws_bytes(ci, co, 27))
    L.check(lib.vc_conv_dgrad_tc(dob.data_ptr(), w.data_ptr(), rb.nbr_bwd.data_ptr(), din.data_ptr(), n, ci, co, 27, 0,
                                 ws.data_ptr(), ws.numel(), _err().data_ptr(), _st()), 'vc_conv_dgrad_tc')
    ref = audit.conv_grads(torch.zeros(n, ci, device=DEV), w.bfloat16().double(), rb.nbr, rb.n_out, dob)[0]
    _note('dgrad_strided', rel_err(din, ref) / TOL['out'], 1, (ci, co, rb.n_out))


@pytest.fixture(scope='module')
def table2d():
    """a many-to-one 2-D table over COUNTS[0] rows: 70 % of the rows on uniform pixels, 30 % on 1 600 hot pixels (~60 rows
    each) -> (nbr [9, n], rep [n])"""
    L, lib = _lib()
    rng = np.random.default_rng(12)
    n = COUNTS[0]
    hot = rng.integers(0, 2 * SHAPE2[0] * SHAPE2[1], 1600)
    pix = np.where(rng.random(n) < 0.7, rng.integers(0, 2 * SHAPE2[0] * SHAPE2[1], n), hot[rng.integers(0, 1600, n)])
    b, r = np.divmod(pix, SHAPE2[0] * SHAPE2[1])
    v, u = np.divmod(r, SHAPE2[1])
    ci = torch.from_numpy(np.stack([b, v, u], 1).astype(np.int32)).to(DEV)
    nbr = torch.empty(9, n, dtype=torch.int32, device=DEV)
    pn = torch.empty(9, dtype=torch.int32, device=DEV)
    rep = torch.empty(n, dtype=torch.int32, device=DEV)
    ws = _ws(lib.vc_subm_rulebook_ws_bytes(n))
    L.check(lib.vc_subm_rulebook_rep(ci.data_ptr(), n, 2, 2, L.host_i32(SHAPE2), L.host_i32([3, 3]), L.host_i32([1, 1]), nbr.data_ptr(),
                                     pn.data_ptr(), rep.data_ptr(), ws.data_ptr(), ws.numel(), _st()), 'vc_subm_rulebook_rep')
    assert int(torch.bincount(rep.long()).max()) >= 48
    return nbr, rep


def _dout_exact_sums(n, c, seed):
    """bf16 output gradients whose per-pixel sums are bf16 values too (small integers times a power of two per column), so
    the gather form's bf16 group sums are exact and the scatter form is the reference for both"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    t = torch.randint(-3, 4, (n, c), device=DEV, generator=g).float()
    scale = torch.pow(2.0, torch.randint(-3, 4, (c,), device=DEV, generator=g).float())
    return (t * scale).bfloat16()


@pytest.mark.parametrize('ci,co', [(16, 16), (16, 32), (32, 32), (32, 64), (64, 64)])
def test_scatter_dgrad(table2d, ctas, ci, co):
    """vc_conv_dgrad_scatter_tc (channels 16 / 32 / 64) on the many-to-one table"""
    L, lib = _lib()
    nbr, _ = table2d
    n = nbr.shape[1]
    w = _weights(ci, co, 9, 400 + ci + co)
    dob = _dout_exact_sums(n, co, 500 + ci)
    din = torch.zeros(n, ci, device=DEV)
    ws = _ws(lib.vc_conv_tc_ws_bytes(ci, co, 9))
    L.check(lib.vc_conv_dgrad_scatter_tc(dob.data_ptr(), w.data_ptr(), nbr.data_ptr(), din.data_ptr(), n, ci, co, 9, ws.data_ptr(),
                                         ws.numel(), _err().data_ptr(), _st()), 'vc_conv_dgrad_scatter_tc')
    ref = audit.conv_grads(torch.zeros(n, ci, device=DEV), w.bfloat16().double(), nbr, n, dob)[0]
    _note('dgrad_scatter', rel_err(din, ref) / TOL['out'], 1, (ci, co))


@pytest.mark.parametrize('ci,co', [(8, 8), (8, 16), (32, 32), (64, 64)])
def test_gather2d_dgrad(table2d, ctas, ci, co):
    """vc_conv_dgrad_gather2d_tc: the same input gradient in gather form (per-pixel sums, one mirrored gather dgrad)"""
    L, lib = _lib()
    nbr, rep = table2d
    n = nbr.shape[1]
    w = _weights(ci, co, 9, 600 + ci + co)
    dob = _dout_exact_sums(n, co, 700 + ci)
    din = torch.full((n, ci), float('nan'), device=DEV)
    ws = _ws(lib.vc_conv_dgrad_gather2d_ws_bytes(n, ci, co, 9))
    L.check(lib.vc_conv_dgrad_gather2d_tc(dob.data_ptr(), w.data_ptr(), nbr.data_ptr(), rep.data_ptr(), din.data_ptr(), n, None, ci,
                                          co, 9, ws.data_ptr(), ws.numel(), _err().data_ptr(), _st()), 'vc_conv_dgrad_gather2d_tc')
    ref = audit.conv_grads(torch.zeros(n, ci, device=DEV), w.bfloat16().double(), nbr, n, dob)[0]
    _note('dgrad_gather2d', rel_err(din, ref) / TOL['out'], 1, (ci, co))


@pytest.mark.parametrize('det', [0, 1])
@pytest.mark.parametrize('training', [1, 0], ids=['train', 'eval'])
@pytest.mark.parametrize('ci,co', [(8, 16), (32, 32), (64, 64)])
def test_conv_bn_relu(coords3, ctas, ci, co, training, det):
    """vc_conv_bn_relu_tc at a device row count of capacity - 77, NaN input rows past it: x, BN statistics, y and the
    running buffers against float64, yb = bf16_rn(y), zero tails of y and yb"""
    L, lib = _lib()
    cap = COUNTS[2]
    n = cap - 77
    nbr = torch.full((27, cap), -1, dtype=torch.int32, device=DEV)
    nbr[:, :n] = _subm(coords3, n)
    w = _weights(ci, co, 27, 800 + ci + co)
    xb = _feats(cap, ci, 900 + ci)
    xb[n:] = float('nan')
    g = torch.Generator(device=DEV).manual_seed(co)
    gamma = 0.5 + torch.rand(co, device=DEV, generator=g)
    beta = 0.1 * torch.randn(co, device=DEV, generator=g)
    rm0 = 0.1 * torch.randn(co, device=DEV, generator=g)
    rv0 = 0.5 + torch.rand(co, device=DEV, generator=g)
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.zeros(1, dtype=torch.int64, device=DEV)
    eps, mom = 1e-3, 0.01
    x = torch.full((cap, co), float('nan'), device=DEV)
    y = torch.full((cap, co), float('nan'), device=DEV)
    yb = torch.full((cap, co), float('nan'), dtype=torch.bfloat16, device=DEV)
    stats = torch.empty(4, co, device=DEV)
    nd = torch.tensor([n], dtype=torch.int32, device=DEV)
    ws = _ws(lib.vc_conv_bn_relu_tc_ws_bytes(cap, ci, co, 27))
    L.check(lib.vc_conv_bn_relu_tc(xb.data_ptr(), w.data_ptr(), nbr.data_ptr(), x.data_ptr(), cap, nd.data_ptr(), ci, co, 27, det,
                                   gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr(), nbt.data_ptr(), mom, eps,
                                   training, y.data_ptr(), co, yb.data_ptr(), co, stats.data_ptr(), ws.data_ptr(), ws.numel(),
                                   _err().data_ptr(), _st()), 'vc_conv_bn_relu_tc')
    torch.cuda.synchronize()
    where = (ci, co, training, det)
    _note('bn_x', rel_err(x[:n], audit.conv(xb[:n], w.bfloat16().double(), nbr, n)) / TOL['out'], 1, where)
    for t in (y, yb):
        assert bool((t[n:] == 0).all()), where
    assert bool(x[n:].isnan().all()), where       # x (read back by the BN backward below the count only): no row past it written
    if training:
        mean, invstd, _, var_u = audit.batch_stats(x[:n], eps)
        want_rm, want_rv = audit.running_update(rm0, rv0, mean, var_u, mom)
        _note('bn_running', max(rel_err(rm, want_rm), rel_err(rv, want_rv)) / TOL['running'], 1, where)
    else:
        mean, invstd = rm0.double(), 1.0 / torch.sqrt(rv0.double() + eps)
        assert torch.equal(rm, rm0) and torch.equal(rv, rv0), where
    assert int(nbt.item()) == training, where
    _note('bn_mean', rel_err(stats[2], mean) / TOL['mean'], 1, where)
    _note('bn_invstd', rel_err(stats[3], invstd) / TOL['invstd'], 1, where)
    _note('bn_y', rel_err(y[:n], audit.bn_relu_fwd(x[:n], mean, invstd, gamma, beta)) / TOL['y'], 1, where)
    assert torch.equal(yb[:n], y[:n].bfloat16()), where
