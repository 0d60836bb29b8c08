"""GPU tests of the device-drawn StVD layer discard (csrc/stvd_layer.cu, the executor's DISCARD op, discard_rng='device'):
the selection bit for bit against the numpy oracle, and every executor mode (exact, static under GraphedStep, phased under
PipelinedStep, VirConv8x's virtual-point stream) against the per-operator module path fed the lists the device drew."""
import copy

import numpy as np
import pytest
import torch

from oracle import stvd_layer as osl
from oracle.testing import fill_module, rel_err

pytestmark = pytest.mark.gpu
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG8 = dict(CFG, LAYER_DISCARD_RATE=0.15, MM=True)
KEYS = ('x_conv1', 'x_conv2', 'x_conv3', 'x_conv4', 'out')
DEV = torch.device('cuda:0')


def _model(precision='fp32'):
    from virconv_b200.backbone import VirConvL8x
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], discard_mode='paper', discard_rng='device', precision=precision)
    fill_module(m, 666)
    return m.to(DEV).train()


def _batch(ids, n_lidar=4096, n_virtual=9000, max_voxels=7000):
    from virconv_b200 import scenes
    b = scenes.make_batch(ids, n_lidar=n_lidar, n_virtual=n_virtual, max_voxels=max_voxels, training=True)
    return {'voxel_features': torch.from_numpy(b.voxel_features.copy()).to(DEV),
            'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).to(DEV), 'batch_size': b.batch_size, 'calib': b.calib,
            'aug_param': torch.from_numpy(b.aug_param.copy())}


def _named(out):
    named = dict(out['multi_scale_3d_features'])
    named['out'] = out['encoded_spconv_tensor']
    return named


def _loss(out):
    from virconv_b200.graph import masked_mean
    return sum(masked_mean(t) for t in _named(out).values())


def _valid(lists):
    """Recorded lists -> exact-length device tensors (static mode: capacity-sized with the count in .num_rows)."""
    out = []
    for t in lists:
        n = getattr(t, 'num_rows', None)
        out.append((t if n is None else t[:int(n)]).clone())
    return out


def _module_step(model, batch, kept):
    """Per-operator module path fed the given kept rows -> (loss, grads, named)."""
    for p in model.parameters():
        p.grad = None
    bd = dict(batch)
    bd['stvd_keep_rows'] = kept
    out = model(bd)
    loss = _loss(out)
    loss.backward()
    torch.cuda.synchronize()
    return float(loss.detach()), {k: v.grad.clone() for k, v in model.named_parameters()}, _named(out)


def _grad_close(got, ref):
    """The bf16 criterion of test_gpu_graph.py: relative L2 below 1e-2, largest difference below 3e-2 of the largest element."""
    got, ref = got.double().cpu(), ref.double().cpu()
    return float((got - ref).norm() / ref.norm().clamp_min(1e-30)) < 1e-2 and rel_err(got.float(), ref.float()) < 3e-2


def _err_flag():
    from virconv_b200 import ops
    return int(ops.tc_error_flag(DEV).item())


# ------------------------------------------------------------------------------------------------ the selection itself
@pytest.mark.parametrize('n', [0, 1, 2, 31, 32, 33, 1023, 1024, 4097, 100003, 215437])
def test_selection_bit_identical_to_oracle(lib_built, n):
    from virconv_b200 import ops
    for rate in (0.1, 0.15, 0.5):
        for seed in (0, 12345, -987654321987):
            s = torch.tensor([seed], dtype=torch.int64, device=DEV)
            want = osl.keep_rows(n, rate, 2, seed)
            k = want.shape[0]
            pos_want = np.full(n, -1)
            pos_want[want] = np.arange(k)
            keep, kept, pos = ops.stvd_layer_keep(n, rate, 2, seed=s)
            assert int(kept) == k, (n, rate, seed)
            assert np.array_equal(keep[:k].cpu().numpy(), want), (n, rate, seed)
            assert bool((keep[k:] == -1).all()) and np.array_equal(pos.cpu().numpy(), pos_want)
            # static form: n valid rows of a larger capacity
            cap = n + 777
            keep2, kept2, pos2 = ops.stvd_layer_keep(cap, rate, 2, seed=s, n_dev=torch.tensor([n], dtype=torch.int32, device=DEV))
            assert int(kept2) == k
            assert np.array_equal(keep2[:k].cpu().numpy(), want) and bool((keep2[k:] == -1).all())
            assert np.array_equal(pos2[:n].cpu().numpy(), pos_want) and bool((pos2[n:] == -1).all())


def test_selection_with_tied_keys(lib_built):
    from virconv_b200 import ops
    rng = np.random.default_rng(4)
    for n, hi in ((8, 6), (5000, 4), (70001, 3), (4097, 1)):
        keys = rng.integers(0, hi, size=n).astype(np.uint32)
        keys[::7] = 0xFFFFFFFF
        for rate in (0.1, 0.37, 0.9):
            want = osl.keep_rows(n, rate, 0, 0, keys=keys)
            keep, kept, _ = ops.stvd_layer_keep(n, rate, 0, keys=torch.from_numpy(keys.astype(np.int64)).to(DEV))
            assert int(kept) == want.shape[0] and np.array_equal(keep[:int(kept)].cpu().numpy(), want), (n, rate)


# ------------------------------------------------------------------------------------------------ exact mode
@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_exact_mode_matches_module_path(lib_built, precision):
    """VirConvL8x paper + 'device' through the plan executor, forward and backward, against the module path fed the lists
    the device drew: indices bit-equal, features within 1e-4, parameter gradients at test_gpu_backbone.py's tolerances."""
    from virconv_b200 import executor
    model = _model(precision)
    twin = copy.deepcopy(model)
    batch = _batch([11, 12])
    for p in model.parameters():
        p.grad = None
    bd = dict(batch)
    out = model(bd)
    assert executor.last_run(model) is not None                # ran through the executor
    named = _named(out)
    loss = _loss(out)
    loss.backward()
    torch.cuda.synchronize()
    assert _err_flag() == 0
    kept = bd['stvd_kept_rows']
    assert len(kept) == 3
    n_in = [batch['voxel_features'].shape[0]]
    for t in kept:
        assert t.dtype == torch.int32 and bool((t[1:] > t[:-1]).all())
    assert kept[0].shape[0] == int(n_in[0] * 0.9)
    ml, mg, mn = _module_step(twin, batch, _valid(kept))
    for k in KEYS:
        assert torch.equal(named[k].indices, mn[k].indices), k
        assert rel_err(named[k].features.detach().cpu(), mn[k].features.detach().cpu()) < 1e-4, k
    assert abs(float(loss) - ml) < 1e-5 * max(1.0, abs(ml))
    for name, p in model.named_parameters():
        if precision == 'bf16':
            assert _grad_close(p.grad, mg[name]), name
        else:
            assert rel_err(p.grad.cpu(), mg[name].cpu()) < 2e-4, name
    # each published tensor's indice_dict only holds rulebooks over its own rows
    d = named['x_conv1'].indice_dict
    assert 'subm1vir1' not in d and 'spvir2' in d and 'subm1vir2' in d
    assert d['spvir2'].nbr_bwd.shape[1] == named['x_conv1'].indices.shape[0]      # built over x_conv1's (kept) rows
    # the eval forward does not discard
    model.eval()
    with torch.no_grad():
        ev = dict(batch)
        model(ev)
    assert 'stvd_kept_rows' not in ev and _named(ev)['x_conv1'].features.shape[0] == n_in[0]


def test_draws_follow_torch_seed_and_stvd_seed(lib_built):
    model = _model('bf16')
    batch = _batch([13, 14])

    def lists(**extra):
        bd = dict(batch)
        bd.update(extra)
        with torch.no_grad():
            model(bd)
        return [t.clone() for t in bd['stvd_kept_rows']]

    torch.manual_seed(5)
    a = lists()
    torch.manual_seed(5)
    b = lists()
    torch.manual_seed(6)
    c = lists()
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert not torch.equal(a[0], c[0])
    seed = torch.tensor([42], dtype=torch.int64, device=DEV)
    d, e = lists(stvd_seed=seed), lists(stvd_seed=seed)
    assert all(torch.equal(x, y) for x, y in zip(d, e))
    n0 = batch['voxel_features'].shape[0]                      # vir_conv1 keeps the input rows: site 0 draws over n0
    assert np.array_equal(d[0].cpu().numpy(), osl.keep_rows(n0, 0.1, 0, 42))


def test_tiny_inputs(lib_built):
    """One input row keeps none after vir_conv1 (int(1 * 0.9) = 0): exact mode refuses naming the site; static mode
    yields zero-row outputs."""
    from virconv_b200 import _lib, executor, ops
    model = _model('bf16')
    b = _batch([15, 16])
    one = dict(b, voxel_features=b['voxel_features'][:1].contiguous(), voxel_coords=b['voxel_coords'][:1].contiguous())
    with pytest.raises(_lib.VirConvLibraryError, match='site 0'):
        with torch.no_grad():
            model(dict(one))
    cap = 256
    vf = torch.zeros((cap, 8), device=DEV)
    vc = torch.full((cap, 4), -1, dtype=torch.int32, device=DEV)
    vf[:1], vc[:1] = one['voxel_features'], one['voxel_coords']
    plan = model._plan()
    caps = {i_out: 256 for _, (_, _, i_in, i_out) in plan.rb_keys.items() if i_out != i_in and i_out != 0}
    spec = executor.StaticSpec(torch.ones(1, dtype=torch.int32, device=DEV), caps, torch.zeros(1, dtype=torch.int32, device=DEV))
    bd = dict(one, voxel_features=vf, voxel_coords=vc, virconv_static=spec,
              virconv_proj=ops.projection_params(one['calib'], one['aug_param'], 2, DEV))
    with torch.no_grad():
        model(bd)
    torch.cuda.synchronize()
    named = _named(bd)
    for k in KEYS:
        assert int(named[k].num_rows.item()) == 0, k
    assert [int(t.num_rows.item()) for t in bd['stvd_kept_rows']] == [0, 0, 0]


def test_virconv8x_mm_stream_matches_module_path(lib_built):
    from virconv_b200 import _lib, scenes
    from virconv_b200.backbone import VirConv8x
    batch = scenes.make_batch_mm([2, 7], n_lidar=4096, n_virtual=6000, max_voxels=3000, training=True)
    m = VirConv8x(CFG8, 8, [1408, 1600, 80], discard_mode='paper', discard_rng='device')
    fill_module(m, 667)
    m.to(DEV).train()
    twin = copy.deepcopy(m)
    res = []
    kept = None
    for model in (m, twin):
        for p in model.parameters():
            p.grad = None
        bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in batch.arrays.items()}
        bd.update(batch_size=2, calib=batch.calib, aug_param=torch.from_numpy(batch.aug_param))
        if kept is not None:
            bd['stvd_keep_rows'] = kept
        out = model(bd)
        if kept is None:
            kept = _valid(bd['stvd_kept_rows'])
            assert len(kept) == 4 and kept[0].shape[0] == int(batch.arrays['voxel_features_mm'].shape[0] * (1 - 0.15))
        pub = {f'{g}:{k}': t for g in ('multi_scale_3d_features', 'multi_scale_3d_features_mm') for k, t in out[g].items()}
        sum(t.features.mean() for t in pub.values()).backward()
        torch.cuda.synchronize()
        res.append((pub, {k: v.grad.clone() for k, v in model.named_parameters()}))
    (pp, pg), (mp, mg) = res
    for k in pp:
        assert torch.equal(pp[k].indices, mp[k].indices), k
        assert rel_err(pp[k].features.detach().cpu(), mp[k].features.detach().cpu()) < 1e-4, k
    for name in pg:
        assert rel_err(pg[name].cpu(), mg[name].cpu()) < 2e-4, name
    one = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in batch.arrays.items()}
    one['voxel_features_mm'] = one['voxel_features_mm'][:1].contiguous()
    one['voxel_coords_mm'] = one['voxel_coords_mm'][:1].contiguous()
    one.update(batch_size=2, calib=batch.calib, aug_param=torch.from_numpy(batch.aug_param))
    with pytest.raises(_lib.VirConvLibraryError, match='site 0'):
        with torch.no_grad():
            m(one)


# ------------------------------------------------------------------------------------------------ captured steps
def _snapshot(holder):
    return _valid(holder['kept'])


def test_graphed_step_fresh_draw_per_replay(lib_built):
    """>= 5 replays over rotating batches: every replay draws new lists, and its loss and gradients are those of the module
    path fed that replay's lists (fp32 kernels: a tolerance that bf16 rounding noise would not allow).  Then a batch beyond
    the (deliberately tight) capacities forces a re-capture."""
    from virconv_b200.graph import GraphedStep
    model = _model('fp32')
    twin = copy.deepcopy(model)
    batches = [_batch([20 + 2 * i, 21 + 2 * i]) for i in range(3)]
    holder = {}

    def loss_fn(out):
        holder['kept'] = out['stvd_kept_rows']
        return _loss(out)

    step = GraphedStep(model, loss_fn, margin=1.35, grain=256)
    params = dict(model.named_parameters())
    got = []
    for s in range(6):
        loss = step(batches[s % 3])
        torch.cuda.synchronize()
        got.append((float(loss), {k: v.grad.clone() for k, v in params.items()}, _snapshot(holder)))
    assert _err_flag() == 0 and step.recaptures == 1
    for s in range(6):
        l, g, kept = got[s]
        if s >= 3:
            assert not torch.equal(kept[0], got[s - 3][2][0]), s              # same batch, new draw
        ml, mg, _ = _module_step(twin, batches[s % 3], kept)
        assert abs(l - ml) < 1e-5 * max(1.0, abs(ml)), s
        for k in params:
            assert rel_err(g[k].cpu(), mg[k].cpu()) < 2e-4, (s, k)
    small = _batch([31, 32], n_lidar=2048, n_virtual=3000, max_voxels=2500)
    big = _batch([33, 34])
    step = GraphedStep(model, loss_fn, margin=1.05, grain=64)
    step(small)
    loss = step(big)                       # more rows than the buffers hold -> re-capture
    torch.cuda.synchronize()
    assert step.recaptures == 2
    ml, _, _ = _module_step(twin, big, _snapshot(holder))
    assert abs(float(loss) - ml) < 1e-5 * max(1.0, abs(ml))


def test_pipelined_step_matches_module_path(lib_built):
    from virconv_b200.graph import PipelinedStep
    model = _model('fp32')
    twin = copy.deepcopy(model)
    batches = [_batch([40 + 2 * i, 41 + 2 * i]) for i in range(3)]
    store, cur = {}, {}

    def loss_fn(out):
        store[cur['inst']] = out['stvd_kept_rows']        # the last call of a capture is the captured graph's
        return _loss(out)

    step = PipelinedStep(model, loss_fn, margin=1.35, grain=256)
    params = dict(model.named_parameters())
    for s in range(5):
        cur['inst'] = s & 1
        loss = step(batches[s % 3])
        torch.cuda.synchronize()
        kept = _valid(store[s & 1])
        l, g = float(loss), {k: v.grad.clone() for k, v in params.items()}
        ml, mg, _ = _module_step(twin, batches[s % 3], kept)
        assert abs(l - ml) < 1e-5 * max(1.0, abs(ml)), s
        for k in params:
            assert rel_err(g[k].cpu(), mg[k].cpu()) < 2e-4, (s, k)
    assert _err_flag() == 0
