"""Chained strided convs composed (vc_set_index_order(1), csrc/rulebook.cu header) against the per-level path (0) on the
same inputs: every index set, device row count, neighbour table (nbr / nbr_bwd), pair count and -1 tail of a forward must be
bit-identical, in exact and static mode, and so must a whole deterministic training step captured in a graph.  Each
comparison also checks that the composed pass ran: 4 (L - 1) launches fewer per chain of L strided convs (one mark, scan and
emit instead of L of each)."""
import pytest
import torch

from oracle.testing import fill_module

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG8 = dict(CFG, LAYER_DISCARD_RATE=0.15, MM=True)


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


def _batch(ids, drop_scene=None, **kw):
    from virconv_b200 import scenes
    b = scenes.make_batch(ids, training=True, **kw)
    keep = slice(None) if drop_scene is None else b.voxel_coords[:, 0] != drop_scene
    return {'voxel_features': torch.from_numpy(b.voxel_features[keep].copy()).to(DEV),
            'voxel_coords': torch.from_numpy(b.voxel_coords[keep].copy()).to(DEV), 'batch_size': b.batch_size, 'calib': b.calib,
            'aug_param': torch.from_numpy(b.aug_param.copy())}


def _snapshot(run):
    """every index set (with its device row count in static mode) and rulebook of a forward, copied out of its arena"""
    from virconv_b200 import executor
    out = {}
    for row in run.plan.rows_i:
        if row[0] == executor.OP_CONV_RB:
            idx, shape = run.indices(row[3])
            out['idx%d' % row[3]] = (idx.clone(), tuple(shape))
            n_dev = run.query(2, row[3])[6]
            if n_dev:
                out['n%d' % row[3]] = executor._view(run.arena, n_dev, (1,), torch.int32).clone()
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


def _saved(*runs):
    """launches the composed pass saves over the per-level path in these runs' plans (no layer discard in them: all the
    strided convs of a plan form one chain)"""
    from virconv_b200 import executor
    return sum(4 * (sum(1 for r in run.plan.rows_i if r[0] == executor.OP_CONV_RB) - 1) for run in runs)


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


@pytest.mark.parametrize('zdim', [80, 40])                # sparse grids [81, 1600, 1408] and [41, 1600, 1408]
@pytest.mark.parametrize('ids', [[3], [5, 6], [7, 8, 9]])
def test_exact_mode_chain_matches_per_level(order, monkeypatch, zdim, ids):
    model = _model(zdim)
    bd = _batch(ids)
    order(0)
    run, n0 = _forward(model, bd, monkeypatch)
    ref = _snapshot(run)
    order(1)
    run, n1 = _forward(model, bd, monkeypatch)
    _equal(ref, _snapshot(run))
    assert sum(1 for k in ref if k.startswith('idx')) == 4
    assert n0 - n1 == _saved(run) == 12


def test_virconv_t_plans_chain_matches_per_level(order, monkeypatch):
    """VirConv-T's training forward: the LiDAR plan and the virtual-point plan each compose their chain"""
    from virconv_b200 import scenes
    from virconv_b200.backbone import VirConv8x
    m = VirConv8x(CFG8, 8, [1408, 1600, 80], precision='bf16')
    fill_module(m, 667)
    m.to(DEV).train()
    b = scenes.make_batch_mm([3, 4], max_voxels=3000, training=True, n_lidar=4096, n_virtual=6000)
    bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
    bd.update(batch_size=b.batch_size, calib=b.calib, aug_param=torch.from_numpy(b.aug_param.copy()))
    order(0)
    runs, n0 = _forward(m, bd, monkeypatch, n_runs=2)
    ref = [_snapshot(r) for r in runs]
    order(1)
    runs, n1 = _forward(m, bd, monkeypatch, n_runs=2)
    for r, s in zip(runs, ref):
        _equal(s, _snapshot(r))
    assert n0 - n1 == _saved(*runs) > 12     # (the LiDAR plan's chain of four and the virtual-point plan's own)


def test_empty_scene(order, monkeypatch):
    model = _model(40)
    bd = _batch([11, 12], drop_scene=0)    # scene 0 has no voxel
    order(0)
    ref = _snapshot(_forward(model, bd, monkeypatch)[0])
    order(1)
    _equal(ref, _snapshot(_forward(model, bd, monkeypatch)[0]))


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
def test_static_mode_chain_matches_per_level(order, monkeypatch, shrink):
    """capacities with head-room, and below the true count of the first or the last strided conv: the clamped counts and the
    overflow value are today's (where the first level overflows, the levels after it count from its whole set: only the
    first level and the flag are compared then)"""
    from virconv_b200 import executor
    model = _model(40)
    bd = _batch([5, 6])
    order(0)
    run, _ = _forward(model, bd, monkeypatch)
    caps = executor.measured_caps(run, 1.3, 256)
    true = executor.measured_caps(run, 1.0, 1)
    keys = sorted(caps)
    if shrink is not None:
        k = keys[0] if shrink == 'first' else keys[-1]
        caps[k] = true[k] - 100
    res = {}
    for mode in (0, 1):
        order(mode)
        sbd, spec = _static_bd(bd, caps)
        run, launches = _forward(model, sbd, monkeypatch)
        res[mode] = (_snapshot(run), int(spec.overflow.item()), launches)
    (ref, ovf_ref, n0), (got, ovf, n1) = res[0], res[1]
    assert n0 - n1 == _saved(run) == 12
    assert ovf == ovf_ref == (0 if shrink is None else true[k])
    if shrink == 'first':
        assert torch.equal(ref['n%d' % keys[0]], got['n%d' % keys[0]]) and int(got['n%d' % keys[0]]) == caps[keys[0]]
        assert torch.equal(ref['idx%d' % keys[0]][0], got['idx%d' % keys[0]][0])
    else:
        _equal(ref, got)
        if shrink == 'last':
            assert int(got['n%d' % keys[-1]]) == caps[keys[-1]]


def _grads_of_step(model_fn, batch, loss_fn, steps=3):
    from virconv_b200.graph import GraphedStep
    m = model_fn()
    step = GraphedStep(m, loss_fn)
    params = dict(m.named_parameters())
    for _ in range(steps):
        loss = step(batch)
    torch.cuda.synchronize()
    return loss.detach().clone(), {k: v.grad.clone() for k, v in params.items()}


def test_graphed_step_bit_identical_in_every_order(order):
    """deterministic mode: a captured VirConv-L training step gives the same loss and gradients, bit for bit, with the index
    composed (1) as one conv after the other (0)"""
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
    torch.use_deterministic_algorithms(True)
    try:
        res = {}
        for mode in (0, 1):
            order(mode)
            res[mode] = _grads_of_step(model_fn, batch, loss_fn)
    finally:
        torch.use_deterministic_algorithms(prev)
    l0, g0 = res[0]
    assert torch.equal(l0, res[1][0])
    for k in g0:
        assert torch.equal(g0[k], res[1][1][k]), k
