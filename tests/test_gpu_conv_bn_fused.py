"""BatchNorm + ReLU inside the tensor-core conv forward (vc_set_conv_bn_fused): the fused launch against the conv followed by
the apply kernel — per layer through the C ABI, and whole training steps of the plan executor (exact mode, a captured
GraphedStep, VirConv8x's two streams with device-drawn StVD).  In deterministic mode the two give the same bits."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle.testing import fill_module, rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG8 = dict(CFG, LAYER_DISCARD_RATE=0.15, MM=True)


def _lib():
    from virconv_b200 import _lib as L
    return L, L.load()


def _err():
    from virconv_b200 import ops
    return ops.tc_error_flag(DEV)


@pytest.fixture
def det_mode():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


def _fused(flag):
    _lib()[1].vc_set_conv_bn_fused(flag)


@pytest.fixture(autouse=True)
def _restore_flag():
    yield
    _fused(int(os.environ.get('VIRCONV_CONV_BN_FUSED', '1') != '0'))


# ------------------------------------------------------------------------------------------------ one layer, C ABI
def _layer(lib, L, c, det, training, n, n_dev, ld, col, inputs):
    from virconv_b200 import ops
    xb, w, nbr, gamma, beta = inputs
    rm = torch.linspace(-0.5, 0.5, c, device=DEV)
    rv = torch.linspace(0.5, 2.0, c, device=DEV)
    nbt = torch.zeros(1, dtype=torch.int64, device=DEV)
    x = torch.empty(n, c, device=DEV)
    y = torch.full((n, ld), 7.0, device=DEV)
    yb = torch.full((n, ld), 7.0, dtype=torch.bfloat16, device=DEV)
    stats = torch.empty(4, c, device=DEV)
    ws = torch.empty(lib.vc_conv_bn_relu_tc_ws_bytes(n, c, c, 27), dtype=torch.uint8, device=DEV)
    nd = torch.tensor([n_dev], dtype=torch.int32, device=DEV) if n_dev is not None else None
    L.check(lib.vc_conv_bn_relu_tc(xb.data_ptr(), w.data_ptr(), nbr.data_ptr(), x.data_ptr(), n, ops._p(nd), c, c, 27, det,
                                   gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr(), nbt.data_ptr(), 0.01, 1e-3,
                                   training, y[:, col:].data_ptr(), ld, yb[:, col:].data_ptr(), ld, stats.data_ptr(),
                                   ws.data_ptr(), ws.numel(), _err().data_ptr(), ops._stream()), 'vc_conv_bn_relu_tc')
    torch.cuda.synchronize()
    rows = n if n_dev is None else n_dev
    return {'x': x[:rows], 'y': y, 'yb': yb, 'stats': stats, 'rm': rm, 'rv': rv, 'nbt': nbt}


@pytest.mark.parametrize('det', [1, 0])
@pytest.mark.parametrize('ctas', [2, 1])
@pytest.mark.parametrize('c', [8, 16, 32, 64])
def test_conv_bn_relu_layer(lib_built, c, ctas, det):
    """dense output, a concat slice (row pitch 2c + 8, column offset 8), a device row count of 0 and one below the capacity
    (tail rows zeroed), BN in training and eval mode"""
    from virconv_b200 import ops
    L, lib = _lib()
    rng = np.random.default_rng(c)
    shape = [20, 100, 100]
    co = np.stack([rng.integers(0, 2, 30000)] + [rng.integers(0, s, 30000) for s in shape], 1).astype(np.int32)
    co = np.unique(co, axis=0)
    rng.shuffle(co)
    n = co.shape[0]
    rb = ops.build_subm_rulebook(torch.from_numpy(np.ascontiguousarray(co)).to(DEV), 2, shape, 3)
    torch.manual_seed(c)
    inputs = (torch.randn(n, c, device=DEV).to(torch.bfloat16), 0.2 * torch.randn(c, 27, c, device=DEV), rb.nbr,
              1 + 0.1 * torch.randn(c, device=DEV), 0.1 * torch.randn(c, device=DEV))
    cases = [(1, None, c, 0), (1, None, 2 * c + 8, 8), (1, 0, c, 0), (1, n - 1000, c, 0), (0, n - 1000, 2 * c + 8, 8)]
    L.check(lib.vc_conv_tc2_config(ctas), 'vc_conv_tc2_config')
    try:
        for training, n_dev, ld, col in cases:
            got = []
            for flag in (1, 0):
                _fused(flag)
                got.append(_layer(lib, L, c, det, training, n, n_dev, ld, col, inputs))
            a, b = got
            assert int(_err().item()) == 0
            case = (training, n_dev, ld, col)
            if n_dev is not None:     # static-mode tail: zeros from the count on, in the slice only
                assert bool((a['y'][n_dev:, col:col + c] == 0).all()) and bool((a['yb'][n_dev:, col:col + c] == 0).all()), case
            assert bool((a['y'][:, :col] == 7).all()) and bool((a['y'][:, col + c:] == 7).all()), case
            assert int(a['nbt'].item()) == training
            for k in a:
                if det or not training or k == 'nbt' or a[k].numel() == 0:
                    assert torch.equal(a[k], b[k]), (case, k)
                else:             # (float64 atomics in another order: the last bits of the sums may differ)
                    assert rel_err(a[k].float().cpu(), b[k].float().cpu()) < 1e-4, (case, k)
    finally:
        lib.vc_conv_tc2_config(0)


# ------------------------------------------------------------------------------------------------ whole steps
def _batch(ids, n_lidar=4096, n_virtual=9000, max_voxels=7000):
    from virconv_b200 import scenes
    b = scenes.make_batch(ids, n_lidar=n_lidar, n_virtual=n_virtual, max_voxels=max_voxels, training=True)
    return {'voxel_features': torch.from_numpy(b.voxel_features.copy()).to(DEV),
            'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).to(DEV), 'batch_size': b.batch_size, 'calib': b.calib,
            'aug_param': torch.from_numpy(b.aug_param.copy())}


def _published(out, groups):
    pub = {}
    for g in groups:
        v = out[g]
        for k, t in (v.items() if isinstance(v, dict) else [('', v)]):
            if t is not None:
                pub[f'{g}:{k}'] = t
    return pub


def _record(model, pub):
    rec = {}
    for k, t in pub.items():
        rec['f:' + k] = t.features.detach().clone()
        rec['i:' + k] = t.indices.clone()
        if getattr(t, 'features_bf16', None) is not None:
            rec['h:' + k] = t.features_bf16.detach().clone()
    rec.update({'g:' + k: v.grad.clone() for k, v in model.named_parameters()})
    rec.update({'b:' + k: v.clone() for k, v in model.named_buffers()})
    return rec


def _same(a, b):
    assert a.keys() == b.keys()
    bad = {k: float((a[k].double() - b[k].double()).abs().max()) for k in a if not torch.equal(a[k], b[k])}
    assert not bad, bad


def test_virconv_l_exact_bit_identical(lib_built, det_mode):
    from virconv_b200.backbone import VirConvL8x
    from virconv_b200.graph import masked_mean
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], precision='bf16')
    fill_module(m, 666)
    m.to(DEV).train()
    state = copy.deepcopy(m.state_dict())
    batch = _batch([3, 4])
    recs = []
    for flag in (1, 0):
        _fused(flag)
        m.load_state_dict(state)
        for p in m.parameters():
            p.grad = None
        pub = _published(m(dict(batch)), ('multi_scale_3d_features', 'encoded_spconv_tensor'))
        sum(masked_mean(t) for t in pub.values()).backward()
        torch.cuda.synchronize()
        recs.append(_record(m, pub))
    assert int(_err().item()) == 0
    _same(*recs)


def test_graphed_step_bit_identical(lib_built, det_mode):
    """the flag is read at capture: one GraphedStep per arm, replayed; features (capacity-sized, zero / -1 tails), gradients,
    BN buffers; and the fused capture launches fewer kernels"""
    from virconv_b200.backbone import VirConvL8x
    from virconv_b200.graph import GraphedStep, masked_mean
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], precision='bf16')
    fill_module(m, 666)
    m.to(DEV).train()
    state = copy.deepcopy(m.state_dict())
    batch = _batch([5, 6])
    recs, launches = [], []
    for flag in (1, 0):
        _fused(flag)
        m.load_state_dict(state)
        pubs = {}

        def loss_fn(out):
            pubs.clear()
            pubs.update(_published(out, ('multi_scale_3d_features', 'encoded_spconv_tensor')))
            return sum(masked_mean(t) for t in pubs.values())

        step = GraphedStep(m, loss_fn)
        for _ in range(3):
            m.load_state_dict(state)
            step(batch)
        torch.cuda.synchronize()
        rec = _record(m, pubs)
        for k, t in pubs.items():
            nr = int(t.num_rows.item())
            assert bool((t.features[nr:] == 0).all()) and bool((t.indices[nr:] == -1).all()), k
        recs.append(rec)
        launches.append(step.launches_per_replay)
        del step
    assert int(_err().item()) == 0
    _same(*recs)
    assert launches[0] < launches[1], launches


def test_virconv8x_paper_stvd_bit_identical(lib_built, det_mode):
    from virconv_b200 import scenes
    from virconv_b200.backbone import VirConv8x
    batch = scenes.make_batch_mm([2, 7], n_lidar=4096, n_virtual=6000, max_voxels=3000, training=True)
    m = VirConv8x(CFG8, 8, [1408, 1600, 80], discard_mode='paper', discard_rng='device', precision='bf16')
    fill_module(m, 667)
    m.to(DEV).train()
    state = copy.deepcopy(m.state_dict())
    recs = []
    for flag in (1, 0):
        _fused(flag)
        m.load_state_dict(state)
        for p in m.parameters():
            p.grad = None
        bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in batch.arrays.items()}
        bd.update(batch_size=2, calib=batch.calib, aug_param=torch.from_numpy(batch.aug_param),
                  stvd_seed=torch.tensor([1234], dtype=torch.int64, device=DEV))
        pub = _published(m(bd), ('multi_scale_3d_features', 'multi_scale_3d_features_mm'))
        sum(t.features.mean() for t in pub.values()).backward()
        torch.cuda.synchronize()
        recs.append(_record(m, pub))
    assert int(_err().item()) == 0
    _same(*recs)
