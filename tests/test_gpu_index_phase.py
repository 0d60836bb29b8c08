"""The plan executor's index phase against the CPU oracle, op by op: for every strided conv (OP_CONV_RB), submanifold rulebook
(OP_SUBM_RB) and projection (OP_INDEX2UV) of a forward, the output index set, device row count, neighbour tables (nbr /
nbr_bwd), pair counts and -1 tails must equal oracle.crulebook / oracle.index2uv applied to the oracle's own inputs, bit for
bit.  Each forward also counts the library's launches, so that a silent fall-back from the composed chain and the batched
index work to per-stage launches fails."""
import numpy as np
import pytest
import torch

from oracle import crulebook as crb
from oracle import index2uv as ouv
from oracle.testing import fill_module

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG8 = dict(CFG, LAYER_DISCARD_RATE=0.15, MM=True)

# Library launches of one bf16 training forward, exact or static mode.  VirConv-L's plan (four NRConv blocks, conv_out):
# stage 1's 3-D rulebook, projection and 2-D rulebook one call each (hash insert + probe, index2uv, hash insert + probe: 5);
# the chain of the four strided convs composed (mark, local scan, block scan, emit: 4) and their tables in one launch (1);
# stages 2-4's 3-D rulebooks, projections and 2-D rulebooks one launch per kind (2 + 1 + 2); 20 fused conv + BatchNorm
# layers; the weight images (1) and the input's bf16 cast (1).
LAUNCHES_L = 5 + 4 + 1 + 5 + 20 + 2
# VirConv-T: the LiDAR plan (stage 1's 3-D rulebook 2, chain of four 4 + 1, stages 2-4's 3-D rulebooks 2, 12 layers, 2)
# and the virtual-point plan (VirConv-L's without conv_out: a chain of three, 19 layers)
LAUNCHES_T = (2 + 4 + 1 + 2 + 12 + 2) + (5 + 4 + 1 + 5 + 19 + 2)
# deterministic mode: stages 2-4's 2-D rulebooks one batch per op, for their `rep` rows (6 launches instead of 2), and the
# row groups of the gather-form dgrad for each of the four 2-D rulebooks (gather2d_prep_dev: 6 launches each)
LAUNCHES_L_DET = LAUNCHES_L + 4 + 4 * 6
# paper-mode StVD: a layer discard after vir_conv1..3 ends a chain, so vir_conv2's and vir_conv3's down convs are chains of
# one and vir_conv4's down conv and conv_out a chain of two.  Stage 1's index work as in LAUNCHES_L (5); per chain its
# count and emit (mark, two scans, emit: 4) and its tables (1), plus the chain of two's lookup of level 1's nbr_fwd (1);
# stages 2-4's 3-D rulebook, projection and 2-D rulebook one launch per kind (1 + 1 + 2); per discard site the row
# selection (7) and the gathers of its indices and features (2); 20 layers, the weight images and the input's bf16 cast
LAUNCHES_L_PAPER = 5 + 3 * (4 + 1) + 1 + 3 * (1 + 1 + 2) + 3 * (7 + 2) + 20 + 2


def _runs(monkeypatch):
    """every executor run of a forward, with its input coordinates and the library launches its call enqueued"""
    from virconv_b200 import _lib, executor
    runs, real, lib = [], executor.run_plan, _lib.load()

    def run_plan(plan, feats, coords, *a, **kw):
        l0 = lib.vc_launch_count()
        run, res = real(plan, feats, coords, *a, **kw)
        run.launches = lib.vc_launch_count() - l0
        run.coords0 = coords.clone()        # (the input index set is the caller's tensor, not in the arena)
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


def _forward(model, bd, monkeypatch, n_runs=1):
    """-> the run records of one forward and the library launches it enqueued"""
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
    return runs, launches


def _model(zdim, **kw):
    from virconv_b200.backbone import VirConvL8x
    torch.manual_seed(0)
    return VirConvL8x(CFG, 8, [1408, 1600, zdim], precision='bf16', **kw).to(DEV).train()


def _lin(idx, shape):
    """batch-major linear cell index of each row"""
    key = idx[:, 0].astype(np.int64)
    for d, s in enumerate(shape):
        key = key * s + idx[:, 1 + d]
    return key


def _in_grid(idx, shape, batch):
    """rows a rulebook takes part in (csrc/rulebook.cu index_ok): batch index and coordinates inside the grid"""
    return (idx[:, 0] >= 0) & (idx[:, 0] < batch) & np.all((idx[:, 1:] >= 0) & (idx[:, 1:] < np.asarray(shape)), axis=1)


def _rows(t, rows):
    """a table of indices into rows[...] -> indices into the whole set (-1 stays -1)"""
    return np.append(rows, -1).astype(np.int32)[t]


def _subm(idx, shape, batch, ks, dl):
    """oracle.crulebook.subm_rulebook over the rows inside the grid; a row outside has only its centre entry (itself)"""
    rows = np.flatnonzero(_in_grid(idx, shape, batch))
    sub = crb.subm_rulebook(idx[rows], shape, ks, dl)
    nbr = np.full((sub.shape[0], len(idx)), -1, np.int32)
    nbr[:, rows] = _rows(sub, rows)
    nbr[sub.shape[0] // 2] = np.arange(len(idx))
    return nbr


def _conv(idx, shape, batch, ks, st, pd, dl):
    """oracle.crulebook.conv_rulebook over the rows inside the grid -> (out indices, out shape, nbr_fwd, nbr_bwd)"""
    rows = np.flatnonzero(_in_grid(idx, shape, batch))
    oi, oshape, nf, nb = crb.conv_rulebook(idx[rows], shape, ks, st, pd, dl)
    nbw = np.full((nb.shape[0], len(idx)), -1, np.int32)
    nbw[:, rows] = nb
    return oi, oshape, _rows(nf, rows), nbw


def _padded(a, cols):
    """[K, cols] int32: a in the first columns, the -1 tail after them"""
    out = np.full((a.shape[0], cols), -1, np.int32)
    out[:, :a.shape[1]] = a
    return out


def _equal(got, want, what):
    got = got.cpu().numpy()
    assert got.shape == want.shape and np.array_equal(got, want), what


def _check_run(run, bd, trans=None):
    """Every index op of `run` against the oracle -> the overflow value static mode must report.  Per index set the oracle
    keeps `full`, the whole set, and `held`, the rows the executor holds: the first min(capacity, count) of it.  Composed
    semantics (csrc/rulebook.cu header): a strided conv's output set is built from its input's whole set, its tables and
    every other op from the held rows.  trans: the [B, 3] transform of the run's projections (default bd['aug_param'])."""
    from virconv_b200 import executor
    calibs, batch = bd['calib'], bd['batch_size']

    def count(iset):   # (capacity, count) of an executor index set
        cap = run.query(2, iset)[1]
        n_dev = run.count(iset)
        return cap, cap if n_dev is None else int(n_dev.item())

    held = {0: run.coords0[:count(0)[1]].cpu().numpy()}
    full, shape, overflow = {0: held[0]}, {0: run.query(2, 0)[3:6]}, 0
    for row in run.plan.rows_i:
        kind, a, b, rb, nd = row[0], row[2], row[3], row[4], row[5]
        ks, st, pd, dl = row[6:6 + nd], row[9:9 + nd], row[12:12 + nd], row[15:15 + nd]
        if kind == executor.OP_CONV_RB:
            oi, oshape, _, _ = _conv(full[a], shape[a], batch, ks, st, pd, dl)
            oi_h, _, nf_h, nb_h = _conv(held[a], shape[a], batch, ks, st, pd, dl)
            cap, cnt = count(b)
            assert cnt == min(cap, len(oi)), 'count of index set %d' % b
            if len(oi) > cap:
                overflow = max(overflow, len(oi))
            got, got_shape = run.indices(b)
            assert list(got_shape) == list(oshape), 'shape of index set %d' % b
            want = np.full((cap, 1 + nd), -1, np.int32)
            want[:cnt] = oi[:cnt]
            _equal(got, want, 'index set %d' % b)
            # the held rows' outputs, ranked in the whole output set; outputs past the held ones have no pair
            pos = np.searchsorted(_lin(oi, oshape), _lin(oi_h, oshape)).astype(np.int32)
            nbw = _rows(nb_h, pos)
            nbw[nbw >= cnt] = -1
            nf = np.full((nf_h.shape[0], cap), -1, np.int32)
            keep = pos < cnt
            nf[:, pos[keep]] = nf_h[:, keep]
            nbr, nbr_bwd, pn, _ = run.rulebook(rb)
            _equal(nbr, nf, 'nbr of rulebook %d' % rb)
            _equal(nbr_bwd, _padded(nbw, count(a)[0]), 'nbr_bwd of rulebook %d' % rb)
            _equal(pn, (nbw >= 0).sum(1).astype(np.int32), 'pair counts of rulebook %d' % rb)
            full[b], held[b], shape[b] = oi, oi[:cnt], list(oshape)
        elif kind == executor.OP_SUBM_RB:
            nbr, _, pn, _ = run.rulebook(rb)
            want = _padded(_subm(held[a], shape[a], batch, ks, dl), count(a)[0])
            _equal(nbr, want, 'nbr of rulebook %d' % rb)
            _equal(pn, (want >= 0).sum(1).astype(np.int32), 'pair counts of rulebook %d' % rb)
        elif kind == executor.OP_INDEX2UV:
            assert (row[22], row[23]) == (1400, 600)   # the oracle's pixel clamp
            uv = ouv.index2uv(held[a], batch, calibs, row[21], bd['aug_param'].numpy() if trans is None else trans)
            _equal(run.indices(b)[0][:len(uv)], uv, 'projection %d' % b)
            full[b] = held[b] = uv
            shape[b] = [row[6], row[7]]
        elif kind == executor.OP_DISCARD:   # (the rows a layer discard keeps: test_gpu_stvd_layer)
            full[b] = held[b] = run.indices(b)[0][:count(b)[1]].cpu().numpy()
            shape[b] = shape[a]
    return overflow


@pytest.mark.parametrize('zdim', [80, 40])                # sparse grids [81, 1600, 1408] and [41, 1600, 1408]
@pytest.mark.parametrize('ids', [[3], [5, 6], [7, 8, 9]])
def test_exact_mode(monkeypatch, zdim, ids):
    bd = _batch(ids)
    runs, launches = _forward(_model(zdim), bd, monkeypatch)
    assert _check_run(runs[0], bd) == 0
    assert launches == LAUNCHES_L


def test_empty_scene(monkeypatch):
    bd = _batch([11, 12], drop_scene=0)    # scene 0 has no voxel
    runs, launches = _forward(_model(40), bd, monkeypatch)
    _check_run(runs[0], bd)
    assert launches == LAUNCHES_L


def test_virconv_t_plans(monkeypatch):
    """VirConv-T's training forward: the LiDAR plan and the virtual-point plan"""
    from virconv_b200 import scenes
    from virconv_b200.backbone import VirConv8x
    m = VirConv8x(CFG8, 8, [1408, 1600, 80], precision='bf16')
    fill_module(m, 667)
    m.to(DEV).train()
    b = scenes.make_batch_mm([3, 4], max_voxels=3000, training=True, n_lidar=4096, n_virtual=6000)
    bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
    bd.update(batch_size=b.batch_size, calib=b.calib, aug_param=torch.from_numpy(b.aug_param.copy()))
    runs, launches = _forward(m, bd, monkeypatch, n_runs=2)
    for run in runs:
        _check_run(run, bd)
    assert launches == LAUNCHES_T


def _launches_no_discard(plan):
    """Library launches of one forward of a plan without layer discards, from its ops: the first stage's submanifold rulebook
    (hash insert + probe: 2), the chain of its strided convs composed (4) with their tables in one launch (1), the later
    stages' submanifold rulebooks one launch per kind (2), one fused conv + BatchNorm launch per layer, the weight images
    and the input's bf16 cast (2).  A plan with projections (index2uv, 2-D rulebooks) is counted by LAUNCHES_L / _T."""
    from virconv_b200 import executor
    kinds = [r[0] for r in plan.rows_i]
    assert executor.OP_INDEX2UV not in kinds and executor.OP_DISCARD not in kinds
    n_conv, n_subm = kinds.count(executor.OP_CONV_RB), kinds.count(executor.OP_SUBM_RB)
    assert n_conv >= 1 and n_subm >= 2
    return 2 + (4 + 1) + 2 + len(plan.layers) + 2


def test_virconv_t_eval_rot3_packed_grid(monkeypatch):
    """VirConv-T's test-time forward at bench.py's eval_rot3 size: the LiDAR plan over the ROT_NUM = 3 copies of 40 000 voxels
    packed along x into [81, 1600, 4 * 1408].  Its input rows are in concat order — copy, then scene — so not batch-contiguous
    as the training input is; every table must still equal the oracle's.  Then each copy's virtual-point plan, its
    projections under that copy's transform."""
    from virconv_b200 import parallel, scenes
    from virconv_b200.backbone import VirConv8x
    m = VirConv8x(CFG8, 8, [1408, 1600, 80], precision='bf16')
    fill_module(m, 667)
    m.to(DEV).eval()
    R = 3
    b = scenes.make_batch_mm(parallel.shard_scene_ids(100, 0, 1, 2), 16384, 80000, 40000, training=False, rot_num=R)
    bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
    bd.update(batch_size=b.batch_size, calib=b.calib, transform_param=torch.from_numpy(b.transform_param.copy()))
    runs, _ = _forward(m, bd, monkeypatch, n_runs=1 + R)
    lidar = runs[0]
    assert lidar.plan is m._plan_lidar()
    W = m.sparse_shape[2]
    assert lidar.query(2, 0)[3:6] == [m.sparse_shape[0], m.sparse_shape[1], 4 * W]
    c = lidar.coords0.cpu().numpy()
    assert len(c) == sum(bd['voxel_coords' + s].shape[0] for s in ['', '1', '2'])
    copy_of = c[:, 3] // W
    assert np.all(np.diff(copy_of) >= 0) and set(copy_of.tolist()) == set(range(R))
    assert np.any(np.diff(c[:, 0]) < 0)               # scene 1 of copy 0 comes before scene 0 of copy 1
    assert _check_run(lidar, bd) == 0
    assert lidar.launches == _launches_no_discard(lidar.plan)
    tp = bd['transform_param'].numpy()
    for i, run in enumerate(runs[1:]):
        assert run.plan is m._plan_mm()
        _check_run(run, bd, tp[:, i])


def test_paper_stvd_chains_of_one_and_two(monkeypatch):
    """VirConv-L's paper-mode StVD discards rows after vir_conv1..3: the strided convs are built as chains of one, one, two"""
    bd = dict(_batch([5, 6]), stvd_seed=torch.tensor([1234], dtype=torch.int64, device=DEV))
    runs, launches = _forward(_model(40, discard_mode='paper', discard_rng='device'), bd, monkeypatch)
    from virconv_b200 import executor
    assert sum(1 for r in runs[0].plan.rows_i if r[0] == executor.OP_DISCARD) == 3
    _check_run(runs[0], bd)
    assert launches == LAUNCHES_L_PAPER


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
def test_static_mode(monkeypatch, shrink):
    """static mode (the index phase enqueued before the first conv): capacities with head-room, and below the true count of
    the first or the last strided conv — clamped counts, -1 tails and the overflow value"""
    from virconv_b200 import executor
    model = _model(40)
    bd = _batch([5, 6])
    runs, _ = _forward(model, bd, monkeypatch)
    caps = executor.measured_caps(runs[0], 1.3, 256)
    true = executor.measured_caps(runs[0], 1.0, 1)
    keys = sorted(caps)
    if shrink is not None:
        k = keys[0] if shrink == 'first' else keys[-1]
        caps[k] = true[k] - 100
    sbd, spec = _static_bd(bd, caps)
    runs, launches = _forward(model, sbd, monkeypatch)
    ovf = _check_run(runs[0], bd)
    assert int(spec.overflow.item()) == ovf == (0 if shrink is None else true[k])
    assert launches == LAUNCHES_L


def test_deterministic_mode(monkeypatch):
    """deterministic mode: the 2-D rulebooks also write the gather-form dgrad's `rep` rows"""
    bd = _batch([5, 6])
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs, launches = _forward(_model(40), bd, monkeypatch)
    finally:
        torch.use_deterministic_algorithms(prev)
    _check_run(runs[0], bd)
    assert launches == LAUNCHES_L_DET
