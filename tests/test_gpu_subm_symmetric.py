"""The plan executor builds the submanifold tables of duplicate-free (3-D) index sets from half the kernel offsets and
mirrors the other half (nbr[k, i] = j exactly when nbr[K-1-k, j] = i).  Every such table of a VirConv-L forward at the
bench's density must equal the full probe of vc_subm_rulebook, neighbour for neighbour and pair
count for pair count."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])


def _runs(monkeypatch):
    from virconv_b200 import executor
    runs, real = [], executor.run_plan

    def run_plan(plan, *a, **kw):
        run, res = real(plan, *a, **kw)
        runs.append(run)
        return run, res

    monkeypatch.setattr(executor, 'run_plan', run_plan)
    return runs


def _batch(ids):
    from virconv_b200 import scenes
    b = scenes.make_batch(ids, training=True)
    return {'voxel_features': torch.from_numpy(b.voxel_features.copy()).to(DEV),
            'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).to(DEV), 'batch_size': b.batch_size, 'calib': b.calib,
            'aug_param': torch.from_numpy(b.aug_param.copy())}


def _check_tables(run, coords0, batch_size):
    """-> number of duplicate-free submanifold tables compared"""
    from virconv_b200 import executor, ops
    checked = 0
    for row in run.plan.rows_i:
        if row[0] != executor.OP_SUBM_RB or not row[21]:
            continue
        nbr, _, pn, meta = run.rulebook(row[4])
        p, n, ndim, s0, s1, s2 = run.query(2, row[2])[:6]
        idx = coords0 if row[2] == 0 else executor._view(run.arena, p, (n, 1 + ndim), torch.int32).clone()
        ref = ops.build_subm_rulebook(idx, batch_size, [s0, s1, s2][:ndim], row[6:6 + ndim], row[15:15 + ndim])
        torch.cuda.synchronize()
        assert meta['unique'] and tuple(nbr.shape) == tuple(ref.nbr.shape)
        assert torch.equal(nbr, ref.nbr), f'table {row[4]}: neighbours differ from the full probe'
        assert torch.equal(pn, ref.pair_num), f'table {row[4]}: pair counts differ from the full probe'
        assert int(ref.pair_num.sum()) > n, 'the table has no neighbours besides the centre offset'
        checked += 1
    return checked


def test_mirrored_subm_tables_match_full_probe(monkeypatch):
    from virconv_b200.backbone import VirConvL8x
    runs = _runs(monkeypatch)
    torch.manual_seed(0)
    model = VirConvL8x(CFG, 8, [1408, 1600, 80], precision='bf16').to(DEV).train()
    bd = _batch([5, 6])
    with torch.no_grad():
        model(bd)
    torch.cuda.synchronize()
    assert len(runs) == 1 and runs[0].static is None
    coords0 = bd['voxel_coords'].to(torch.int32).contiguous()
    assert _check_tables(runs[0], coords0, bd['batch_size']) >= 4
