"""GPU tests of the captured test-time forward: the x-batching kernels (vc_xbatch_pack / vc_xbatch_split) and the row-counted
consumers of static tensors (vc_dense_rows_f32, vc_voxel2pinds_rows) bit for bit against the numpy restatement and the
existing kernels, and graph.GraphedForward against the eager eval forward of VirConv-T (ROT_NUM = 3 and 1) and VirConv-L."""
import numpy as np
import pytest
import torch

from oracle import xbatch as oxb
from oracle.testing import fill_module, rel_err

pytestmark = pytest.mark.gpu
CFG8 = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.15, NUM_FILTERS=[16, 32, 64, 64], MM=True)
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
DEV = torch.device('cuda:0')
KW = dict(n_lidar=4096, n_virtual=6000)
MAX_VOXELS = 3000
VOX = dict(point_cloud_range=(0, -40, -3, 70.4, 40, 1), voxel_size=(0.05, 0.05, 0.05), max_points_per_voxel=5,
           max_voxels=MAX_VOXELS, vfe_model='max', max_voxels_mm=MAX_VOXELS, vfe_model_mm=None)


@pytest.fixture(autouse=True)
def _no_pipeline_timeout(lib_built):
    """Every test leaves the tensor-core kernels' pipeline-timeout flag at 0."""
    yield
    from virconv_b200 import ops
    torch.cuda.synchronize()
    assert int(ops.tc_error_flag(DEV).item()) == 0


# -- kernels ------------------------------------------------------------------------------------------------------
def _split_case(rng, n, cap, C, W, xs):
    f = np.full((cap, C), np.nan, dtype=np.float32)
    idx = np.full((cap, 4), -1, dtype=np.int32)
    f[:n] = rng.standard_normal((n, C)).astype(np.float32)
    idx[:n] = np.stack([rng.integers(0, 2, n), rng.integers(0, 3, n), rng.integers(0, 40, n), rng.choice(xs, n)], 1)
    if cap > n:
        idx[n:n + (cap - n) // 2, 3] = W // 8              # garbage past the count that looks like a copy-0 row
    return f, idx


@pytest.mark.parametrize('C', [16, 32, 64])
def test_xbatch_split_matches_oracle(C):
    from virconv_b200 import ops
    rng = np.random.default_rng(C)
    W = 4 * 50
    q = W // 4
    every = list(range(0, W))
    cases = {
        'boundaries': (3000, 3584, [0, 1, q - 1, q, q + 1, 2 * q, 2 * q + 1, 3 * q - 1, 3 * q, 3 * q + 1, 4 * q - 1]),
        'empty copy': (2000, 2304, [x for x in every if not (q < x < 2 * q)]),
        'one copy': (1500, 1536, list(range(2 * q + 1, 3 * q))),
        'count = capacity': (1024, 1024, every),
        'nothing valid': (0, 512, every),
        'tile edge': (257, 700, every),
    }
    for R in (1, 3, 4):
        for name, (n, cap, xs) in cases.items():
            f, idx = _split_case(rng, n, cap, C, W, xs)
            got = ops.xbatch_split(torch.from_numpy(f).to(DEV), torch.from_numpy(idx).to(DEV),
                                   torch.tensor([n], dtype=torch.int32, device=DEV), W, R)
            want = oxb.split(f, idx, n, W, R)
            assert len(got) == R
            for i, ((gf, gi, gn), (wf, wi, wn)) in enumerate(zip(got, want)):
                assert int(gn) == wn, (R, name, i)
                assert torch.equal(gi.cpu(), torch.from_numpy(wi)), (R, name, i)
                assert torch.equal(gf.cpu(), torch.from_numpy(wf)), (R, name, i)      # bit for bit, zero tail
    with pytest.raises(ValueError, match='1..4'):
        ops.xbatch_split(torch.zeros(4, C, device=DEV), torch.zeros(4, 4, dtype=torch.int32, device=DEV),
                         torch.zeros(1, dtype=torch.int32, device=DEV), W, 5)


def test_xbatch_split_rejects_bad_arguments_in_the_library():
    from virconv_b200 import _lib
    lib = _lib.load()
    p = _lib.host_ptrs([0] * 5)
    assert lib.vc_xbatch_split(None, None, 0, None, 16, 200, 5, p, p, p, None, 0, None) == -1       # R > 4: VC_ERR_INVALID
    assert lib.vc_xbatch_split(None, None, 0, None, 8, 200, 2, p, p, p, None, 0, None) == -4        # C = 8: unsupported
    assert lib.vc_xbatch_pack(p, p, p, _lib.host_i32([0] * 5), 5, 8, 10, 0, None, None, None, None) == -1


def test_xbatch_pack_matches_cat():
    """Against torch.cat of the exact rows with x += i*W; NaN / garbage rows past every copy's count; an empty copy."""
    from virconv_b200 import ops
    rng = np.random.default_rng(3)
    W = 176
    for ns in ((900, 0, 1300), (5,), (700, 800, 900, 1000)):
        feats, coords, counts, exact_f, exact_c = [], [], [], [], []
        for i, n in enumerate(ns):
            cap = n + 77
            f = torch.full((cap, 8), float('nan'))
            c = torch.full((cap, 4), 9, dtype=torch.int32)
            f[:n] = torch.from_numpy(rng.standard_normal((n, 8)).astype(np.float32))
            c[:n] = torch.from_numpy(np.stack([rng.integers(0, 2, n), rng.integers(0, 41, n), rng.integers(0, 1600, n),
                                               rng.integers(0, W, n)], 1).astype(np.int32))
            feats.append(f.to(DEV))
            coords.append(c.to(DEV))
            counts.append(torch.tensor([n], dtype=torch.int32, device=DEV))
            exact_f.append(f[:n])
            exact_c.append(c[:n] + torch.tensor([0, 0, 0, i * W], dtype=torch.int32))
        pf, pc, tot = ops.xbatch_pack(feats, coords, counts, W)
        n = sum(ns)
        assert int(tot) == n and pf.shape[0] == sum(f.shape[0] for f in feats)
        assert torch.equal(pf[:n].cpu(), torch.cat(exact_f)) and torch.equal(pc[:n].cpu(), torch.cat(exact_c))
        assert bool((pf[n:] == 0).all()) and bool((pc[n:] == -1).all())
        of, oc, on = oxb.pack([f.cpu().numpy() for f in feats], [c.cpu().numpy() for c in coords], list(ns), W)
        assert on == n and np.array_equal(pf.cpu().numpy(), of) and np.array_equal(pc.cpu().numpy(), oc)


def _static_tensor(rng, n, cap, C, shape, B):
    """A static-mode tensor: n unique coordinates in `shape`, garbage features and a -1 index tail past the count."""
    cells = rng.choice(B * int(np.prod(shape)), n, replace=False)
    b, rest = np.divmod(cells, int(np.prod(shape)))
    z, rest = np.divmod(rest, shape[1] * shape[2])
    y, x = np.divmod(rest, shape[2])
    idx = np.full((cap, 4), -1, dtype=np.int32)
    idx[:n] = np.stack([b, z, y, x], 1)
    f = np.full((cap, C), 1.0e30, dtype=np.float32)
    f[:n] = rng.standard_normal((n, C)).astype(np.float32)
    return torch.from_numpy(f).to(DEV), torch.from_numpy(idx).to(DEV)


def test_dense_rows_and_voxel2pinds_rows_on_a_static_tensor():
    """The row-counted kernels on a static tensor equal the existing kernels on its exact rows; the -1 tail writes nothing
    (guard regions before and after the outputs unchanged); the dense() gradient of the tail rows is zero."""
    from virconv_b200 import _lib, ops
    from virconv_b200 import spconv_compat as spconv
    lib = _lib.load()
    rng = np.random.default_rng(11)
    B, C, shape = 2, 16, [3, 20, 24]
    n, cap = 900, 1280
    f, idx = _static_tensor(rng, n, cap, C, shape, B)
    cnt = torch.tensor([n], dtype=torch.int32, device=DEV)
    spatial = int(np.prod(shape))
    guard = C * spatial + shape[1] * shape[2] + shape[2] + 64        # reach of a (-1, -1, -1, -1) row below the output
    buf = torch.full((guard + B * C * spatial + guard,), 7.0, device=DEV)
    body = buf[guard:guard + B * C * spatial]
    body.zero_()
    _lib.check(lib.vc_dense_rows_f32(f.data_ptr(), idx.data_ptr(), cap, cnt.data_ptr(), C, 3, B, _lib.host_i32(shape),
                                     body.data_ptr(), ops._stream()), 'vc_dense_rows_f32')
    ref = spconv.SparseConvTensor(f[:n].clone(), idx[:n].clone(), shape, B).dense()
    assert torch.equal(body.view(B, C, *shape), ref)
    assert bool((buf[:guard] == 7.0).all()) and bool((buf[guard + B * C * spatial:] == 7.0).all())
    t = spconv.SparseConvTensor(f.clone().requires_grad_(True), idx, shape, B)
    t.num_rows = cnt
    d = t.dense()                                                   # routes to vc_dense_rows_f32
    assert torch.equal(d, ref)
    g = torch.randn_like(d)
    d.backward(g)
    fe = f[:n].clone().requires_grad_(True)
    spconv.SparseConvTensor(fe, idx[:n].clone(), shape, B).dense().backward(g)
    assert torch.equal(t.features.grad[:n], fe.grad) and bool((t.features.grad[n:] == 0).all())

    gv = spatial + shape[1] * shape[2] + shape[2] + 64
    vbuf = torch.full((gv + B * spatial + gv,), 12345, dtype=torch.int32, device=DEV)
    vbody = vbuf[gv:gv + B * spatial]
    _lib.check(lib.vc_voxel2pinds_rows(idx.data_ptr(), cap, cnt.data_ptr(), 3, B, _lib.host_i32(shape), vbody.data_ptr(),
                                       ops._stream()), 'vc_voxel2pinds_rows')
    vref = ops.voxel2pinds(idx[:n].clone(), B, shape)
    assert torch.equal(vbody.view(B, *shape), vref)
    assert bool((vbuf[:gv] == 12345).all()) and bool((vbuf[gv + B * spatial:] == 12345).all())
    assert torch.equal(ops.voxel2pinds(idx, B, shape, num_rows=cnt), vref)


# -- GraphedForward against the eager eval forward ---------------------------------------------------------------
def _model_t(precision, mm=True):
    from virconv_b200.backbone import VirConv8x
    m = VirConv8x(dict(CFG8, MM=mm), 8, [1408, 1600, 80], precision=precision)
    fill_module(m, 667)
    return m.to(DEV).eval()


def _model_l(precision):
    from virconv_b200.backbone import VirConvL8x
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], precision=precision)
    fill_module(m, 666)
    return m.to(DEV).eval()


def _batch_t(ids, R, max_voxels=MAX_VOXELS, **kw):
    from virconv_b200 import scenes
    b = scenes.make_batch_mm(ids, max_voxels=max_voxels, training=False, rot_num=R, **dict(KW, **kw))
    bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
    bd.update(batch_size=b.batch_size, calib=b.calib, transform_param=torch.from_numpy(b.transform_param.copy()))
    return bd


def _points_t(ids, R, **kw):
    """The same test-time scenes as _batch_t before voxelisation: per copy 'points{i}' (LiDAR) and 'points_mm{i}' (virtual
    points), the reference's keys after X_TRANS.input_transform and the stream split (dataset.py:270-281)."""
    from virconv_b200 import scenes
    kw = dict(KW, **kw)
    out = {'batch_size': len(ids)}
    calibs, clouds = [], {}
    for b, sid in enumerate(ids):
        calib = scenes.Calib()
        calibs.append(calib)
        pts = scenes.make_points(sid, kw['n_lidar'], kw['n_virtual'], calib)
        for i in range(R):
            p = scenes.augment(pts, scenes.TEST_TRANSFORMS[i])
            s = '' if i == 0 else str(i)
            for key, ind in (('points', 2), ('points_mm', 1)):
                q = scenes.mask_points_by_range(p[p[:, 7] == ind], scenes.POINT_CLOUD_RANGE).astype(np.float32)
                clouds.setdefault(key + s, []).append(np.concatenate([np.full((q.shape[0], 1), b, np.float32), q], 1))
    out.update({k: torch.from_numpy(np.concatenate(v)).to(DEV) for k, v in clouds.items()})
    out['calib'] = calibs
    out['transform_param'] = torch.from_numpy(np.tile(scenes.TEST_TRANSFORMS[None, :R], (len(ids), 1, 1)).astype(np.float32))
    return out


def _batch_l(ids, **kw):
    from virconv_b200 import scenes
    b = scenes.make_batch(ids, max_voxels=MAX_VOXELS, training=False, **dict(KW, **kw))
    return {'voxel_features': torch.from_numpy(b.voxel_features).to(DEV), 'voxel_coords': torch.from_numpy(b.voxel_coords).to(DEV),
            'batch_size': b.batch_size, 'calib': b.calib}


def _named(out, R):
    named = {}
    for s in [''] + [str(i) for i in range(1, R)]:
        named['out' + s] = out['encoded_spconv_tensor' + s]
        for g in ('multi_scale_3d_features', 'multi_scale_3d_features_mm'):
            for k, t in out.get(g + s, {}).items():
                if t is not None:
                    named[f'{g}{s}:{k}'] = t
    return named


def _close(got, ref, precision):
    if ref.numel() == 0:
        return got.numel() == 0
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    if precision == 'fp32':
        return rel_err(got, ref) < 1e-5
    # the bf16 criterion of test_gpu_graph_t.py: relative L2 below 1e-2, largest difference below 3e-2 of the largest element
    return float((got - ref).norm() / ref.norm().clamp_min(1e-30)) < 1e-2 and rel_err(got, ref) < 3e-2


def _eager(model, batch, R, bev=False):
    with torch.no_grad():
        out = model(dict(batch))
        named = {k: (t.features.clone(), t.indices.int().clone(), list(t.spatial_shape)) for k, t in _named(out, R).items()}
        dense = {}
        if bev:
            for s in [''] + [str(i) for i in range(1, R)]:
                d = out['encoded_spconv_tensor' + s].dense()
                n, c, dd, h, w = d.shape
                dense[s] = d.view(n, c * dd, h, w).clone()
    torch.cuda.synchronize()
    return named, dense


def _check(got, ref, R, precision, what=''):
    named, dense = ref
    g = _named(got, R)
    assert sorted(g) == sorted(named), what
    for k, (f, idx, shape) in named.items():
        t = g[k]
        rows = int(t.num_rows.item())
        assert t.num_rows.dtype == torch.int32 and t.num_rows.is_cuda, (what, k)
        assert rows == f.shape[0], (what, k, rows, f.shape[0])
        assert list(t.spatial_shape) == shape, (what, k)
        assert torch.equal(t.indices[:rows].int(), idx), (what, k)
        assert _close(t.features[:rows], f, precision), (what, k)
        if t.features.shape[0] > rows:
            assert float(t.features[rows:].abs().max()) == 0.0, (what, k)
            assert bool((t.indices[rows:] == -1).all()), (what, k)
    for s, d in dense.items():
        assert got['spatial_features' + s].shape == d.shape, (what, s)
        assert _close(got['spatial_features' + s], d, precision), (what, s)
        assert got['spatial_features_stride' + s] == 8


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
@pytest.mark.parametrize('case', ['T-rot3', 'T-rot1', 'L'])
def test_graphed_forward_matches_eager(case, precision):
    """Every published tensor of one replay: the eager eval forward's row counts and indices, features within 1e-5 (fp32) or
    the bf16 criterion, zero / -1 tails; with bev=True the spatial features equal the eager .dense().view(...)."""
    from virconv_b200.graph import GraphedForward
    if case == 'L':
        model, batch, R = _model_l(precision), _batch_l([3, 4]), 1
    else:
        R = 3 if case == 'T-rot3' else 1
        model, batch = _model_t(precision), _batch_t([3, 4], R)
    ref = _eager(model, batch, R, bev=True)
    fwd = GraphedForward(model, margin=1.3, bev=True, grain=256)
    out = fwd(batch)
    torch.cuda.synchronize()
    assert fwd.recaptures == 1 and fwd.launches_per_replay > 0
    assert int(fwd.ovf_host.max()) == 0
    _check(out, ref, R, precision, case)
    assert out['calib'] is batch['calib']                             # the batch's own keys pass through


def test_graphed_forward_lidar_only_model():
    """VirConv8x without the virtual-point stream (MM: False): only the packed LiDAR plan is captured."""
    from virconv_b200.graph import GraphedForward
    model, batch = _model_t('bf16', mm=False), _batch_t([7, 8], 2)
    batch = {k: v for k, v in batch.items() if '_mm' not in k}
    ref = _eager(model, batch, 2)
    out = GraphedForward(model, grain=256)(batch)
    torch.cuda.synchronize()
    _check(out, ref, 2, 'bf16', 'lidar only')


def test_replays_over_rotating_batches():
    """9 replays over 4 batches, each against its own eager forward (results read before the next call)."""
    from virconv_b200.graph import GraphedForward
    model = _model_t('bf16')
    batches = [_batch_t([20 + 2 * i, 21 + 2 * i], 3) for i in range(4)]
    refs = [_eager(model, b, 3) for b in batches]
    fwd = GraphedForward(model, margin=1.35, grain=256)
    for s in range(9):
        out = fwd(batches[s % 4])
        _check(out, refs[s % 4], 3, 'bf16', 'replay %d' % s)
    assert fwd.recaptures == 1


def test_in_graph_voxelisers_match_eager_voxelisation():
    """2R vc_voxelize_mean calls inside the graph (max-VFE for LiDAR, plain mean for the virtual points) against the eager
    forward on the host-voxelised batch of the same scenes and transforms."""
    from virconv_b200.graph import GraphedForward
    model = _model_t('bf16')
    ids = [[41, 42], [43, 44]]
    refs = [_eager(model, _batch_t(i, 3), 3) for i in ids]
    fwd = GraphedForward(model, margin=1.35, grain=256, voxelizer=VOX)
    for s in range(4):
        out = fwd(_points_t(ids[s % 2], 3))
        _check(out, refs[s % 2], 3, 'bf16', 'vox %d' % s)
    assert fwd.recaptures == 1
    assert [st.cap0 for st in fwd.streams] == [2 * MAX_VOXELS] * 6


def test_overflow_recaptures_and_returns_the_exact_result(monkeypatch):
    """margin 1.0 sized on a small batch, then a larger one: the call grows the graph and returns the eager result.  Then one
    strided conv's capacity 300 rows short: the replay's flag reports it, the same call re-captures and re-runs the batch."""
    from virconv_b200 import executor
    from virconv_b200.graph import GraphedForward
    model = _model_t('fp32')
    small, large = _batch_t([5, 6], 3, n_lidar=2048, n_virtual=3000), _batch_t([5, 6], 3)
    ref_s, ref_l = _eager(model, small, 3), _eager(model, large, 3)
    fwd = GraphedForward(model, margin=1.0, grain=1)
    _check(fwd(small), ref_s, 3, 'fp32', 'small')
    assert fwd.recaptures == 1
    _check(fwd(large), ref_l, 3, 'fp32', 'large')
    assert fwd.recaptures >= 2

    real = executor.measured_caps
    calls = []

    def tight(run, margin=1.3, grain=1024):          # the first capture's LiDAR plan: first strided set 300 rows short
        c = real(run, margin, grain)
        calls.append(run)
        if len(calls) == 1:
            first = sorted(c)[0]
            c[first] = real(run, 1.0, 1)[first] - 300
        return c

    monkeypatch.setattr(executor, 'measured_caps', tight)
    fwd = GraphedForward(model, margin=1.3, grain=256)
    out = fwd(large)
    torch.cuda.synchronize()
    assert fwd.recaptures == 2
    first = sorted(real(calls[0], 1.0, 1))[0]
    assert fwd.overflow_events == [{'': real(calls[0], 1.0, 1)[first]}]     # the LiDAR plan only, the rows that did not fit
    _check(out, ref_l, 3, 'fp32', 'after overflow')


def test_deterministic_replays_bit_identical():
    """torch.use_deterministic_algorithms(True): two replays of one batch publish bit-identical tensors (tails included)."""
    from virconv_b200.graph import GraphedForward
    model = _model_t('bf16')
    batch = _batch_t([9, 10], 3)
    torch.use_deterministic_algorithms(True)
    try:
        fwd = GraphedForward(model, grain=256, bev=True)
        recs = []
        for _ in range(2):
            out = fwd(batch)
            rec = {k: (t.features.clone(), t.indices.clone(), t.num_rows.clone()) for k, t in _named(out, 3).items()}
            rec.update({'bev' + s: (out['spatial_features' + s].clone(),) for s in ('', '1', '2')})
            recs.append(rec)
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    assert fwd.recaptures == 1
    bad = [k for k in recs[0] if not all(torch.equal(a, b) for a, b in zip(recs[0][k], recs[1][k]))]
    assert not bad, bad
