"""CPU checks of the captured test-time forward (graph.GraphedForward, VirConv8x's static eval forward): what is refused,
and with which error, before anything reaches a device; the per-copy bookkeeping; and the numpy restatement of the device
x-batching (oracle/xbatch.py) against the reference's `decompose_tensor` restated in oracle/backbone.py."""
import numpy as np
import pytest
import torch

CFG8 = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.15, NUM_FILTERS=[16, 32, 64, 64], MM=True)
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])


def _model8(cfg=CFG8):
    from virconv_b200.backbone import VirConv8x
    return VirConv8x(cfg, 8, [1408, 1600, 80]).eval()


def _model_l():
    from virconv_b200.backbone import VirConvL8x
    return VirConvL8x(CFG, 8, [1408, 1600, 80]).eval()


def _spec():
    from virconv_b200 import executor
    return executor.StaticSpec(torch.zeros(1, dtype=torch.int32), {}, torch.zeros(1, dtype=torch.int32))


def _bd(R, mm=True, **extra):
    bd = {'batch_size': 2, 'calib': None}
    if R > 1:
        bd['transform_param'] = torch.zeros(2, R, 3)
    for s in [''] + [str(i) for i in range(1, R)]:
        for p in ('', '_mm') if mm else ('',):
            bd['voxel_features' + p + s] = torch.zeros(4, 8)
            bd['voxel_coords' + p + s] = torch.zeros(4, 4, dtype=torch.int32)
    bd.update(extra)
    return bd


def _eval_spec(R, mm=True):
    from virconv_b200.backbone import EvalStaticSpec
    return EvalStaticSpec(_spec(), [torch.zeros(1, dtype=torch.int32)] * R, [_spec() for _ in range(R)] if mm else [],
                          torch.zeros(R, 2, 28))


def test_graphed_forward_refusals():
    from virconv_b200.graph import GraphedForward
    with pytest.raises(ValueError, match='GraphedStep'):
        GraphedForward(_model8().train())                                   # a training-mode model
    with pytest.raises(ValueError, match='VirConvL8x or VirConv8x'):
        GraphedForward(torch.nn.Linear(2, 2))
    with pytest.raises(ValueError, match='check_overflow'):
        GraphedForward(_model8(), check_overflow='never')
    g = GraphedForward(_model8())
    with pytest.raises(ValueError, match='1..4 transformed copies'):
        g(_bd(5))
    bd = _bd(3)
    del bd['voxel_coords_mm2']
    with pytest.raises(ValueError, match='voxel_coords_mm2'):               # a missing copy key
        g(bd)
    with pytest.raises(ValueError, match="points1, points_mm1"):
        GraphedForward(_model8(), voxelizer={})(dict(_bd(2), points=torch.zeros(1, 9), points_mm=torch.zeros(1, 9)))
    gl = GraphedForward(_model_l())
    with pytest.raises(ValueError, match='VirConvL8x runs one copy'):      # VirConv-L has no X_TRANS
        gl(_bd(3, mm=False))
    assert gl.copies(_bd(1, mm=False)) == 1


def test_old_static_keys_in_eval_still_refused():
    """The training StaticSpecs keep their refusal in an eval forward, also next to the new key."""
    m = _model8()
    with pytest.raises(ValueError, match='training forward only'):
        m(_bd(1, virconv_static=_spec(), virconv_static_mm=_spec()))
    with pytest.raises(ValueError, match='training forward only'):
        m(_bd(3, virconv_static=_spec(), virconv_static_mm=_spec(), virconv_eval_static=_eval_spec(3)))


def test_eval_static_spec_refusals():
    m = _model8()
    with pytest.raises(ValueError, match='1..4 transformed copies'):
        m(_bd(5, virconv_eval_static=_eval_spec(4)))
    with pytest.raises(ValueError, match='describes 2 LiDAR'):
        m(_bd(3, virconv_eval_static=_eval_spec(2)))
    bd = _bd(2, virconv_eval_static=_eval_spec(2))
    del bd['voxel_features1']
    with pytest.raises(ValueError, match='voxel_features1'):
        m(bd)
    spec = _eval_spec(2)
    spec.proj = None
    with pytest.raises(ValueError, match='projection blocks'):
        m(_bd(2, virconv_eval_static=spec))
    with pytest.raises(ValueError, match='test-time forward'):
        _model8().train()(_bd(1, virconv_eval_static=_eval_spec(1)))


def test_per_copy_bookkeeping():
    from virconv_b200.graph import GraphedForward
    g = GraphedForward(_model8())
    assert g.input_streams(3) == ['', '1', '2', '_mm', '_mm1', '_mm2']
    assert g.plan_streams(3) == ['', '_mm', '_mm1', '_mm2']
    assert g.input_streams(1) == ['', '_mm'] and g.plan_streams(1) == ['', '_mm']
    lidar = GraphedForward(_model8(dict(CFG8, MM=False)))
    assert lidar.input_streams(2) == ['', '1'] and lidar.plan_streams(2) == ['']
    gl = GraphedForward(_model_l())
    assert gl.input_streams(1) == [''] and gl.plan_streams(1) == ['']
    assert g.copies(_bd(3)) == 3 and g.copies(_bd(1)) == 1
    # voxeliser settings per stream: every virtual-point copy reads the '_mm' entries; its VFE defaults to the plain mean
    from virconv_b200.graph import _Stream
    vox = dict(point_cloud_range=(0, -40, -3, 70.4, 40, 1), voxel_size=(0.05, 0.05, 0.05), max_points_per_voxel=5,
               max_voxels=40000, vfe_model='max')
    g = GraphedForward(_model8(), voxelizer=dict(vox, max_voxels_mm=30000))
    assert [g._vox_arg(_Stream(s, 0), 'max_voxels') for s in ('', '2', '_mm', '_mm2')] == [40000, 40000, 30000, 30000]
    assert [g._vox_arg(_Stream(s, 0), 'vfe_model') for s in ('1', '_mm1')] == ['max', None]


def _rows(rng, n, xs):
    idx = np.stack([rng.integers(0, 2, n), rng.integers(0, 2, n), rng.integers(0, 50, n), rng.choice(xs, n)], 1).astype(np.int32)
    return rng.standard_normal((n, 16)).astype(np.float32), idx


def test_split_matches_decompose_tensor():
    """Hand-built rows with x at i*q, (i+1)*q, inside the copies and >= R*q, a NaN / -1 garbage tail past the count: the
    restatement keeps exactly the rows decompose_tensor keeps, in order, moved back by i*q."""
    from oracle import spconv_cpu
    from oracle import xbatch
    from oracle.backbone import decompose_tensor
    W, R = 176 * 4, 3
    q = W // 4
    rng = np.random.default_rng(5)
    xs = [0, 1, q - 1, q, q + 1, 2 * q - 1, 2 * q, 2 * q + 5, 3 * q - 1, 3 * q, 3 * q + 1, 4 * q - 1]
    n, cap = 300, 384
    f, idx = _rows(rng, n, xs)
    assert {0, q, 2 * q, 3 * q} <= set(idx[:, 3].tolist())
    fc = np.full((cap, 16), np.nan, dtype=np.float32)
    ic = np.full((cap, 4), -1, dtype=np.int32)
    fc[:n], ic[:n] = f, idx
    ic[n:n + 20, 3] = q + 3                                                  # garbage past the count is never read
    parts = xbatch.split(fc, ic, n, W, R)
    t = spconv_cpu.SparseConvTensor(torch.from_numpy(f), torch.from_numpy(idx), [2, 50, W], 2)
    for i, (pf, pi, k) in enumerate(parts):
        ref = decompose_tensor(t, i, 2)
        assert k == ref.indices.shape[0] and k > 0
        assert np.array_equal(pi[:k], ref.indices.numpy()) and np.array_equal(pf[:k], ref.features.numpy())
        assert (pi[k:] == -1).all() and (pf[k:] == 0).all()
        assert ref.spatial_shape == [2, 50, q]
    kept = sum(p[2] for p in parts)
    assert kept == int(((idx[:, 3] % q != 0) & (idx[:, 3] < R * q)).sum())   # x == i*q and x >= R*q go nowhere


def test_pack_then_split_round_trip():
    """pack is torch.cat of the exact rows with x += i*W; splitting a tensor laid out like it returns each copy."""
    from oracle import xbatch
    rng = np.random.default_rng(7)
    W = 64
    copies = []
    for i, n in enumerate((40, 0, 25)):
        f, idx = _rows(rng, n, list(range(1, W)))
        cap = n + 16
        fc = np.full((cap, 16), np.nan, dtype=np.float32)
        ic = np.full((cap, 4), 7, dtype=np.int32)
        fc[:n], ic[:n] = f, idx
        copies.append((fc, ic, n))
    pf, pc, tot = xbatch.pack([c[0] for c in copies], [c[1] for c in copies], [c[2] for c in copies], W)
    ref_c = np.concatenate([c[1][:c[2]] + np.array([0, 0, 0, i * W], dtype=np.int32) for i, c in enumerate(copies)])
    ref_f = np.concatenate([c[0][:c[2]] for c in copies])
    assert tot == 65 and pf.shape[0] == sum(c[0].shape[0] for c in copies)
    assert np.array_equal(pc[:tot], ref_c) and np.array_equal(pf[:tot], ref_f)
    assert (pc[tot:] == -1).all() and (pf[tot:] == 0).all()
    for i, (f, idx, k) in enumerate(xbatch.split(pf, pc, tot, 4 * W, 3)):
        fc, ic, n = copies[i]
        assert k == n and np.array_equal(idx[:k], ic[:n]) and np.array_equal(f[:k], fc[:n])
