"""The chain-level tables built by lookup in the chain's ranked output bitmaps (csrc/rulebook.cu: subm_lookup_kernel for the
stage 2-4 3-D submanifold rulebooks, conv_fwd_lookup_kernel for the nbr_fwd of the strided convs after the first) against
the CPU oracle, on a small scene whose voxels lie on every face of the grid and at the batch boundary: a neighbour cell
past a face must be rejected per dimension, not by linear-index arithmetic that wraps x = W - 1 onto the next row's x = 0
or scene 0's last cell onto scene 1's first.  In static mode a level whose capacity is below its count holds its first
`capacity` cells only, and no table may point past the rows its index set holds."""
import numpy as np
import pytest
import torch

from test_gpu_index_phase import DEV, LAUNCHES_L, _batch, _check_run, _forward, _model, _static_bd

pytestmark = pytest.mark.gpu
ZDIM = 40


def _block(lo, hi):
    """every cell (z, y, x) of the box lo <= c <= hi"""
    z, y, x = np.meshgrid(*[np.arange(a, b + 1) for a, b in zip(lo, hi)], indexing='ij')
    return np.stack([z.ravel(), y.ravel(), x.ravel()], 1)


def _boundary_batch():
    """Two scenes of a [41, 1600, 1408] grid: per scene, 3 x 3 x 3 blocks in the eight corners and at the centre of each of
    the six faces, and scattered interior cells; scene 0 ends in the grid's last cell, scene 1 starts in its first."""
    bd = _batch([5, 6])
    D, H, W = ZDIM + 1, 1600, 1408
    rng = np.random.default_rng(7)
    cells = []
    for b in range(2):
        pts = []
        for z in (0, D - 3):
            for y in (0, H - 3):
                for x in (0, W - 3):
                    pts.append(_block((z, y, x), (z + 2, y + 2, x + 2)))
        mid = (D // 2 - 1, H // 2 - 1, W // 2 - 1)
        for d, edge in ((0, 0), (0, D - 3), (1, 0), (1, H - 3), (2, 0), (2, W - 3)):
            lo = list(mid)
            lo[d] = edge
            pts.append(_block(lo, [v + 2 for v in lo]))
        pts.append(np.stack([rng.integers(0, D, 800), rng.integers(0, H, 800), rng.integers(0, W, 800)], 1))
        c = np.unique(np.concatenate(pts), axis=0)
        cells.append(np.concatenate([np.full((len(c), 1), b), c], 1))
    coords = np.concatenate(cells).astype(np.float32)
    assert coords[:, 1:].min() == 0 and np.array_equal(coords[:, 1:].max(0), [D - 1, H - 1, W - 1])
    last0 = np.flatnonzero(coords[:, 0] == 0)[-1]
    assert np.array_equal(coords[last0], [0, D - 1, H - 1, W - 1]) and np.array_equal(coords[last0 + 1], [1, 0, 0, 0])
    feats = bd['voxel_features'][torch.arange(len(coords), device=DEV) % bd['voxel_features'].shape[0]]
    return dict(bd, voxel_features=feats, voxel_coords=torch.from_numpy(coords).to(DEV))


def _conv_sets(run):
    """output index-set ids of the strided convs, in plan order"""
    from virconv_b200 import executor
    return [r[3] for r in run.plan.rows_i if r[0] == executor.OP_CONV_RB]


def _held(run, iset):
    n_dev = run.count(iset)
    return run.query(2, iset)[1] if n_dev is None else int(n_dev.item())


def _no_entry_past_held(run):
    """every table entry is -1 or a row its index set holds: nbr / subm tables into the input set, nbr_bwd into the output"""
    from virconv_b200 import executor
    for r in run.plan.rows_i:
        kind, a, b, rb = r[0], r[2], r[3], r[4]
        if kind not in (executor.OP_CONV_RB, executor.OP_SUBM_RB):
            continue
        nbr, nbr_bwd, _, _ = run.rulebook(rb)
        assert int(nbr.max()) < _held(run, a), 'rulebook %d points past the rows of index set %d' % (rb, a)
        if nbr_bwd is not None:
            assert int(nbr_bwd.max()) < _held(run, b), 'nbr_bwd of rulebook %d points past index set %d' % (rb, b)


def test_boundary_exact(monkeypatch):
    bd = _boundary_batch()
    runs, launches = _forward(_model(ZDIM), bd, monkeypatch)
    assert _check_run(runs[0], bd) == 0
    _no_entry_past_held(runs[0])
    assert launches == LAUNCHES_L


@pytest.mark.parametrize('level', [0, 1])
def test_boundary_static_overflow(monkeypatch, level):
    """static mode, the capacity of the chain's level-`level` output set at half its count: the later levels' nbr_fwd and
    the submanifold tables over that set see its held rows only"""
    from virconv_b200 import executor
    model = _model(ZDIM)
    bd = _boundary_batch()
    runs, _ = _forward(model, bd, monkeypatch)
    caps = executor.measured_caps(runs[0], 1.3, 256)
    true = executor.measured_caps(runs[0], 1.0, 1)
    k = _conv_sets(runs[0])[level]
    caps[k] = true[k] // 2
    sbd, spec = _static_bd(bd, caps)
    runs, launches = _forward(model, sbd, monkeypatch)
    assert _held(runs[0], k) == caps[k]
    assert int(spec.overflow.item()) == _check_run(runs[0], bd) >= true[k]
    _no_entry_past_held(runs[0])
    assert launches == LAUNCHES_L
