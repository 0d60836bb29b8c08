"""GPU tests of the device-drawn StVD input front end (csrc/stvd.cu, vc_stvd_input_front_end; preprocess.input_front_end):
rows, order and row counts of every stream bit for bit against the numpy oracle (oracle/stvd_input.py) at bench size, the
static form (capacity, device row count, tails, overflow), the launch count and a captured replay drawing afresh."""
import numpy as np
import pytest
import torch

from oracle import stvd_input as osi

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
PC = (0, -40, -3, 70.4, 40, 1)


def _collated(scene_ids, n_lidar=16384, n_virtual=400000, empty=()):
    from virconv_b200 import scenes
    rows = []
    for b, sid in enumerate(scene_ids):
        p = scenes.make_points(sid, n_lidar, 0 if b in empty else n_virtual)
        rows.append(np.pad(p, ((0, 0), (1, 0)), constant_values=b))
    return np.ascontiguousarray(np.concatenate(rows)).astype(np.float32)


def _check(got, want, later_fusion):
    names = ('points', 'points_mm') if later_fusion else ('points',)
    for name in names:
        g = got[name].cpu().numpy()
        assert g.shape == want[name].shape, (name, g.shape, want[name].shape)
        np.testing.assert_array_equal(got['stvd_input_kept' + name[6:]].cpu().numpy(), want['src_' + name])
        assert g.tobytes() == want[name].tobytes(), name
    np.testing.assert_array_equal(got['stvd_input_status'].cpu().numpy(), want['status'])


@pytest.mark.parametrize('B', [1, 2, 4])
@pytest.mark.parametrize('later_fusion', [False, True])
@pytest.mark.parametrize('training', [True, False])
def test_bit_identical_to_oracle_at_bench_size(lib_built, B, later_fusion, training):
    from virconv_b200 import preprocess
    pts = _collated([3, 4, 5, 6][:B])
    seed = 0x1234_5678_9ABC_DEF0 - B
    bins = 2 if training else 10
    got = preprocess.input_front_end(torch.from_numpy(pts).to(DEV), B, training, later_fusion,
                                     seed=torch.tensor([seed], dtype=torch.int64, device=DEV), point_cloud_range=PC)
    want = osi.front_end(pts, B, bins, 0.8, later_fusion, shuffle=training, seed=seed, pc_range=PC)
    _check(got, want, later_fusion)
    assert int(got['stvd_input_overflow']) == 0


@pytest.mark.parametrize('static', [False, True])
def test_scene_without_virtual_points(lib_built, static):
    from virconv_b200 import preprocess
    pts = _collated([7, 8, 9], n_lidar=4096, n_virtual=20000, empty=(1,))
    seed = 77
    n = pts.shape[0]
    cap = n + 1000
    buf = torch.zeros((cap, pts.shape[1]), dtype=torch.float32, device=DEV)
    buf[:n] = torch.from_numpy(pts).to(DEV)
    buf[n:, 0] = 1                                     # rows past n_dev are never read
    buf[n:, -1] = 2
    n_dev = torch.tensor([n], dtype=torch.int32, device=DEV)
    got = preprocess.input_front_end(buf if static else buf[:n], 3, True, True, seed=torch.tensor([seed], device=DEV),
                                     n_dev=n_dev if static else None, point_cloud_range=PC, static=static)
    want = osi.front_end(pts, 3, 2, 0.8, True, True, seed=seed, pc_range=PC)
    assert want['status'].tolist() == [0, 1, 0]
    if static:
        for name in ('points', 'points_mm'):
            t, k = got[name], got['stvd_input_kept' + name[6:]]
            m = int(t.num_rows)
            assert t.shape[0] == cap and m == want[name].shape[0]
            tail = t[m:].cpu().numpy()
            assert (tail[:, 0] == -1).all() and (tail[:, 1:] == 0).all()
            assert (k[m:] == -1).all()
            got[name], got['stvd_input_kept' + name[6:]] = t[:m], k[:m]
    _check(got, want, True)


def test_overflow_is_flagged(lib_built):
    from virconv_b200 import preprocess
    pts = _collated([3, 4], n_lidar=4096, n_virtual=20000)
    want = osi.front_end(pts, 2, 2, 0.8, True, True, seed=5, pc_range=PC)
    rows = [want['points'].shape[0], want['points_mm'].shape[0]]
    cap = min(rows) - 50
    got = preprocess.input_front_end(torch.from_numpy(pts).to(DEV), 2, True, True, seed=torch.tensor([5], device=DEV),
                                     point_cloud_range=PC, cap=cap, static=True)
    assert int(got['stvd_input_overflow']) == sum(r - cap for r in rows)
    assert int(got['points'].num_rows) == cap and int(got['points_mm'].num_rows) == cap


def test_launches_and_capture_draw_afresh(lib_built):
    from virconv_b200 import _lib, preprocess
    lib = _lib.load()
    pts = torch.from_numpy(_collated([3, 4], n_lidar=4096, n_virtual=20000)).to(DEV)
    preprocess.input_front_end(pts, 2, True, True, static=True)          # warm (workspace, modules)
    torch.cuda.synchronize()
    l0 = lib.vc_launch_count()
    preprocess.input_front_end(pts, 2, True, True, static=True)
    assert lib.vc_launch_count() - l0 == 22
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):                                            # fails on any host read or synchronisation
        out = preprocess.input_front_end(pts, 2, True, True, static=True)
    draws = []
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        m = int(out['points_mm'].num_rows)
        draws.append(out['stvd_input_kept_mm'][:m].sort().values.cpu().numpy())
    assert draws[0].shape == draws[1].shape                              # the same plan ...
    assert not np.array_equal(draws[0], draws[1])                        # ... a fresh subset per replay


def test_independent_draws_per_copy(lib_built):
    from virconv_b200 import preprocess
    pts = _collated([3], n_lidar=2048, n_virtual=20000)
    seed = torch.tensor([11], device=DEV)
    kept = []
    for draw in (0, 1):
        r = preprocess.input_front_end(torch.from_numpy(pts).to(DEV), 1, False, True, seed=seed, draw=draw,
                                       point_cloud_range=PC)
        want = osi.front_end(pts, 1, 10, 0.8, True, False, seed=11, draw=draw, pc_range=PC)
        _check(r, want, True)
        kept.append(want['src_points_mm'])
    assert not np.array_equal(kept[0], kept[1])
