"""Index order 2 (vc_set_index_order(2): the chain's per-stage index work batched into one launch per kind, and in static
mode the index phase before the first feature kernel) against order 1 (the same work one launch per stage) and order 0 on
the same inputs: every index set, device row count, neighbour table (nbr / nbr_bwd), pair count and -1 tail of a forward
must be bit-identical, and so must a deterministic captured training step.  Each comparison also counts the library's
launches, so that a silent fall-back to the per-stage path fails."""
import pytest
import torch

from oracle.testing import fill_module

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG8 = dict(CFG, LAYER_DISCARD_RATE=0.15, MM=True)
# VirConv-L: conv_tables of the four strided convs 4 -> 1, and for the three stages behind vir_conv2..4's down convs the
# 3-D hash insert + probe 6 -> 2, index2uv 3 -> 1, 2-D hash insert + probe 6 -> 2
SAVED_L = 3 + 4 + 2 + 4
SAVED_L_DET = 3 + 4 + 2           # deterministic mode: the 2-D rulebooks (with their `rep` rows) stay per stage


@pytest.fixture
def order():
    from virconv_b200 import _lib
    lib = _lib.load()

    def set_order(mode):
        assert lib.vc_set_index_order(mode) == 0
    yield set_order
    set_order(1)


def _runs(monkeypatch):
    from virconv_b200 import executor
    runs, real = [], executor.run_plan

    def run_plan(plan, *a, **kw):
        run, res = real(plan, *a, **kw)
        runs.append(run)
        return run, res

    monkeypatch.setattr(executor, 'run_plan', run_plan)
    return runs


def _batch(ids, drop_scene=None):
    from virconv_b200 import scenes
    b = scenes.make_batch(ids, training=True)
    keep = slice(None) if drop_scene is None else b.voxel_coords[:, 0] != drop_scene
    return {'voxel_features': torch.from_numpy(b.voxel_features[keep].copy()).to(DEV),
            'voxel_coords': torch.from_numpy(b.voxel_coords[keep].copy()).to(DEV), 'batch_size': b.batch_size, 'calib': b.calib,
            'aug_param': torch.from_numpy(b.aug_param.copy())}


def _snapshot(run, n0=None):
    """every index set (with its device row count in static mode), projection and rulebook of a forward, copied out of its
    arena (n0: the input voxels' count of a static-mode forward)"""
    from virconv_b200 import executor
    out = {}
    for row in run.plan.rows_i:
        if row[0] in (executor.OP_CONV_RB, executor.OP_INDEX2UV):
            idx, shape = run.indices(row[3])
            n = run.query(2, row[3])[1]
            n_dev = run.query(2, row[3])[6]
            if n_dev:   # static mode (a projection's rows past the count are not written; the input voxels' count is the caller's)
                cnt = int(executor._view(run.arena, n_dev, (1,), torch.int32)) if row[2] != 0 else n0
                out['n%d' % row[3]] = cnt
                if row[0] == executor.OP_INDEX2UV:
                    n = cnt
            out['idx%d' % row[3]] = (idx[:n].clone(), tuple(shape))
        if row[0] in (executor.OP_CONV_RB, executor.OP_SUBM_RB):
            nbr, nbw, pn, meta = run.rulebook(row[4])
            out['rb%d' % row[4]] = (nbr.clone(), None if nbw is None else nbw.clone(), None if pn is None else pn.clone(), meta)
    torch.cuda.synchronize()
    return out


def _equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        for x, y in zip(a[k] if isinstance(a[k], tuple) else (a[k],), b[k] if isinstance(b[k], tuple) else (b[k],)):
            if isinstance(x, torch.Tensor):
                assert x.shape == y.shape and torch.equal(x, y), k
            else:
                assert x == y, k


def _forward(model, bd, monkeypatch, n_runs=1):
    """-> the run record(s) of one forward and the library launches it enqueued"""
    from virconv_b200 import _lib
    lib = _lib.load()
    runs = _runs(monkeypatch)
    torch.cuda.synchronize()
    l0 = lib.vc_launch_count()
    with torch.no_grad():
        model(dict(bd))
    torch.cuda.synchronize()
    launches = lib.vc_launch_count() - l0
    assert len(runs) == n_runs
    return (runs[0] if n_runs == 1 else runs), launches


def _model(zdim, seed=0):
    from virconv_b200.backbone import VirConvL8x
    torch.manual_seed(seed)
    return VirConvL8x(CFG, 8, [1408, 1600, zdim], precision='bf16').to(DEV).train()


def _compare(order, model, bd, monkeypatch, modes=(0, 1, 2), n_runs=1):
    res = {}
    for mode in modes:
        order(mode)
        runs, launches = _forward(model, bd, monkeypatch, n_runs)
        runs = runs if n_runs > 1 else [runs]
        res[mode] = ([_snapshot(r) for r in runs], launches)
    for mode in modes[1:]:
        for a, b in zip(res[modes[0]][0], res[mode][0]):
            _equal(a, b)
    return {m: r[1] for m, r in res.items()}


@pytest.mark.parametrize('zdim', [80, 40])                # sparse grids [81, 1600, 1408] and [41, 1600, 1408]
@pytest.mark.parametrize('ids', [[3], [5, 6], [7, 8, 9]])
def test_exact_mode_batched_matches(order, monkeypatch, zdim, ids):
    n = _compare(order, _model(zdim), _batch(ids), monkeypatch)
    assert n[1] - n[2] == SAVED_L


def test_empty_scene(order, monkeypatch):
    n = _compare(order, _model(40), _batch([11, 12], drop_scene=0), monkeypatch)    # scene 0 has no voxel
    assert n[1] - n[2] == SAVED_L


def test_virconv_t_plans(order, monkeypatch):
    """VirConv-T's training forward: the LiDAR plan and the virtual-point plan each batch their chain's stages"""
    from virconv_b200 import scenes
    from virconv_b200.backbone import VirConv8x
    m = VirConv8x(CFG8, 8, [1408, 1600, 80], precision='bf16')
    fill_module(m, 667)
    m.to(DEV).train()
    b = scenes.make_batch_mm([3, 4], max_voxels=3000, training=True, n_lidar=4096, n_virtual=6000)
    bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
    bd.update(batch_size=b.batch_size, calib=b.calib, aug_param=torch.from_numpy(b.aug_param.copy()))
    n = _compare(order, m, bd, monkeypatch, n_runs=2)
    assert n[1] - n[2] > SAVED_L


def test_paper_stvd_falls_back(order, monkeypatch):
    """VirConv-L's paper-mode StVD discards rows after vir_conv1..3: no chain of strided convs, so order 2 launches exactly
    what order 1 does"""
    from virconv_b200.backbone import VirConvL8x
    torch.manual_seed(0)
    m = VirConvL8x(CFG, 8, [1408, 1600, 40], discard_mode='paper', discard_rng='device', precision='bf16').to(DEV).train()
    bd = dict(_batch([5, 6]), stvd_seed=torch.tensor([1234], dtype=torch.int64, device=DEV))
    n = _compare(order, m, bd, monkeypatch, modes=(1, 2))
    assert n[1] == n[2]


def _static_bd(bd, caps, margin=1.25):
    from virconv_b200 import executor, ops
    n = bd['voxel_features'].shape[0]
    cap0 = (int(n * margin) + 255) // 256 * 256
    vf = torch.zeros((cap0, bd['voxel_features'].shape[1]), device=DEV)
    vc = torch.full((cap0, 4), -1.0, device=DEV)
    vf[:n] = bd['voxel_features']
    vc[:n] = bd['voxel_coords']
    spec = executor.StaticSpec(torch.tensor([n], dtype=torch.int32, device=DEV), caps, torch.zeros(1, dtype=torch.int32, device=DEV))
    out = dict(bd, voxel_features=vf, voxel_coords=vc, virconv_static=spec,
               virconv_proj=ops.projection_params(bd['calib'], bd['aug_param'], bd['batch_size'], DEV))
    return out, spec


@pytest.mark.parametrize('shrink', [None, 'first', 'last'])
def test_static_mode_batched_matches(order, monkeypatch, shrink):
    """static mode (order 2 enqueues the index phase first): capacities with head-room, and below the true count of the
    first or the last strided conv — the same clamped counts, tails and overflow value as order 1"""
    from virconv_b200 import executor
    model = _model(40)
    bd = _batch([5, 6])
    order(1)
    run, _ = _forward(model, bd, monkeypatch)
    caps = executor.measured_caps(run, 1.3, 256)
    true = executor.measured_caps(run, 1.0, 1)
    keys = sorted(caps)
    if shrink is not None:
        k = keys[0] if shrink == 'first' else keys[-1]
        caps[k] = true[k] - 100
    res = {}
    for mode in (1, 2):
        order(mode)
        sbd, spec = _static_bd(bd, caps)
        run, launches = _forward(model, sbd, monkeypatch)
        res[mode] = (_snapshot(run, bd['voxel_features'].shape[0]), int(spec.overflow.item()), launches)
    (ref, ovf_ref, n1), (got, ovf, n2) = res[1], res[2]
    _equal(ref, got)
    assert ovf == ovf_ref == (0 if shrink is None else true[k])
    assert n1 - n2 == SAVED_L


def test_deterministic_forward_keeps_2d_rep(order, monkeypatch):
    """deterministic mode: the 2-D rulebooks keep their per-stage probe (it writes the gather-form dgrad's `rep` rows); the
    rest is batched, and every table is the same"""
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        n = _compare(order, _model(40), _batch([5, 6]), monkeypatch, modes=(1, 2))
    finally:
        torch.use_deterministic_algorithms(prev)
    assert n[1] - n[2] == SAVED_L_DET


def _step_result(model_fn, batch, loss_fn, steps=3):
    from virconv_b200.graph import GraphedStep
    m = model_fn()
    step = GraphedStep(m, loss_fn)
    params = dict(m.named_parameters())
    for _ in range(steps):
        loss = step(batch)
    torch.cuda.synchronize()
    return loss.detach().clone(), {k: v.grad.clone() for k, v in params.items()}


def _graphed_steps(order, deterministic):
    from virconv_b200.backbone import VirConvL8x
    from virconv_b200.graph import masked_mean
    batch = _batch([5, 6])

    def model_fn():
        m = VirConvL8x(CFG, 8, [1408, 1600, 40], precision='bf16')
        fill_module(m, 666)
        return m.to(DEV).train()

    def loss_fn(out):
        return masked_mean(out['encoded_spconv_tensor']) + sum(masked_mean(t) for t in out['multi_scale_3d_features'].values())

    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        res = {}
        for mode in (1, 2):
            order(mode)
            res[mode] = _step_result(model_fn, batch, loss_fn)
    finally:
        torch.use_deterministic_algorithms(prev)
    return res


def test_graphed_step_deterministic_bit_identical(order):
    """a captured deterministic VirConv-L training step (index phase first, two-CTA conv grids in order 2): the same loss and
    gradients, bit for bit"""
    res = _graphed_steps(order, True)
    assert torch.equal(res[1][0], res[2][0])
    for k in res[1][1]:
        assert torch.equal(res[1][1][k], res[2][1][k]), k


def test_graphed_step_matches(order):
    """the non-deterministic captured step: the loss and the gradients within the bf16 run-to-run spread (fp32 atomics)"""
    res = _graphed_steps(order, False)
    assert torch.allclose(res[1][0], res[2][0], rtol=1e-5, atol=0)
    for k, ref in res[1][1].items():
        got = res[2][1][k].double()
        ref = ref.double()
        assert float((got - ref).norm() / ref.norm().clamp_min(1e-30)) < 1e-2, k
