"""Device-drawn StVD input front end, host side: the numpy oracle (oracle/stvd_input.py) against the reference's own
partition / input_point_discard (tests/golden/stvd_input_plan.npz) and the host path's `_discard_plan`, and the law of its
draws (keep frequencies of a subsampled bin, the shuffle a permutation)."""
import os

import numpy as np
import pytest

from oracle import stvd_input as osi
from virconv_b200 import preprocess

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'stvd_input_plan.npz')


def _golden():
    g = np.load(GOLD)
    return [(str(n), g) for n in g['names']]


@pytest.mark.parametrize('name', [n for n, _ in _golden()])
def test_plan_matches_reference_golden(name):
    g = np.load(GOLD)
    x = g[f'{name}:points'][:, 0]
    bn, position, distant, zero_div = (int(v) for v in g[f'{name}:meta'])
    rate = float(g[f'{name}:rate'])
    b = osi.bins(x, bn)
    counts = np.bincount(b[b >= 0], minlength=bn)
    assert counts[::-1].tolist() == g[f'{name}:before'].tolist()          # parts are far -> near
    if zero_div:
        with pytest.raises(ZeroDivisionError):
            osi.plan(counts, x.shape[0], bn, rate)
        return
    pos, per_bin, out_n, take = osi.plan(counts, x.shape[0], bn, rate)
    assert pos == position
    kept = np.where(take < 0, counts, take)
    assert kept[::-1].tolist() == g[f'{name}:after'].tolist()
    assert out_n == int(x.shape[0] * (1 - rate))
    assert per_bin == int((out_n - distant) / (position + 0.0001))


def test_golden_covers_the_edge_cases():
    seen = set()
    for name, g in _golden():
        bn, position, _, zero_div = (int(v) for v in g[f'{name}:meta'])
        x = g[f'{name}:points'][:, 0]
        before = g[f'{name}:before']
        seen.add(('bins', bn))
        if zero_div:
            seen.add('no virtual points')
            continue
        pos, per_bin, _, _ = osi.plan(before[::-1], x.shape[0], bn, float(g[f'{name}:rate']))
        seen |= {'empty bin'} if (before == 0).any() else set()
        seen |= {'one bin'} if (before > 0).sum() == 1 else set()
        seen |= {'position 0'} if pos == 0 else set()
        seen |= {'per_bin <= 0'} if per_bin <= 0 else set()
        seen |= {'x < 0'} if (x < 0).any() else set()
        seen |= {'NaN'} if np.isnan(x).any() else set()
    assert seen >= {('bins', 2), ('bins', 10), 'no virtual points', 'empty bin', 'one bin', 'position 0', 'per_bin <= 0',
                    'x < 0', 'NaN'}


def test_plan_matches_host_discard_plan():
    rng = np.random.default_rng(0)
    for t in range(3000):
        bn = (2, 10, 7, 16)[t % 4]
        counts = rng.integers(0, rng.choice([3, 50, 5000]), bn)
        if rng.random() < 0.3:
            counts[rng.integers(0, bn)] += rng.integers(0, 100000)
        n_all = int(counts.sum() + rng.integers(0, 20))             # (points in no bin count in n_all)
        if n_all == 0:
            continue
        rate = float(rng.choice([0.8, 0.5, 0.2, 0.95, 0.0, 1.0]))
        _, _, _, take = osi.plan(counts, n_all, bn, rate)
        segs, _, n_out = preprocess._discard_plan(counts, n_all, bn, rate, np.random.RandomState(1))
        got = {b: c for b, _, c, _ in segs}
        want = np.where(take < 0, counts, take)
        assert [got[b] for b in range(bn)] == want.tolist(), (t, counts.tolist(), n_all, rate)
        assert n_out == want.sum()


def _cloud(B, n_lidar, n_virtual, seed=0):
    rng = np.random.default_rng(seed)
    rows = []
    for b in range(B):
        p = np.zeros((n_lidar + n_virtual, 9), np.float32)
        p[:, 0] = b
        p[:, 1] = rng.uniform(-5, 75, p.shape[0])
        p[:, 2] = rng.uniform(-45, 45, p.shape[0])
        p[:, 3:8] = rng.uniform(-1, 1, (p.shape[0], 5))
        p[:, 8] = np.r_[np.full(n_lidar, 2.0), np.ones(n_virtual)]
        rows.append(p[rng.permutation(p.shape[0])])                 # LiDAR and virtual interleaved
    return np.concatenate(rows)


def test_keep_frequency_of_a_subsampled_bin():
    pts = _cloud(1, 0, 300, seed=1)
    x = pts[:, 1]
    b = osi.bins(x, 2)
    counts = np.bincount(b[b >= 0], minlength=2)
    _, _, _, take = osi.plan(counts, pts.shape[0], 2, 0.8)
    sub = [k for k in range(2) if take[k] >= 0]
    assert sub
    hits = np.zeros(pts.shape[0])
    draws = 400
    for seed in range(draws):
        r = osi.front_end(pts, 1, 2, 0.8, later_fusion=True, shuffle=False, seed=seed, pc_range=(-100, -100, -3, 100, 100, 1))
        hits[r['src_points_mm']] += 1
    for k in sub:
        p = take[k] / counts[k]
        f = hits[b == k] / draws
        assert abs(f.mean() - p) < 1e-9                              # exactly take rows per draw
        assert np.abs(f - p).max() < 5 * np.sqrt(p * (1 - p) / draws) + 1e-9
    keep_all = [k for k in range(2) if take[k] < 0]
    for k in keep_all:
        assert (hits[b == k] == draws).all()
    assert (hits[b < 0] == 0).all()


@pytest.mark.parametrize('n', [0, 1, 2, 3, 5, 17, 64, 100, 1000, 4097])
def test_shuffle_is_a_permutation(n):
    for seed in (0, 1, -5):
        p = osi.feistel(np.arange(n), n, 3, 1, seed)
        assert sorted(p.tolist()) == list(range(n))


def test_shuffle_positions_are_uniform():
    n, draws = 7, 3000
    pos = np.array([osi.feistel(np.arange(n), n, 0, 0, s)[0] for s in range(draws)])
    freq = np.bincount(pos, minlength=n) / draws
    assert np.abs(freq - 1 / n).max() < 5 * np.sqrt((1 / n) * (1 - 1 / n) / draws)


@pytest.mark.parametrize('later_fusion', [False, True])
def test_oracle_front_end_assembles_like_the_host_flow(later_fusion):
    """Without shuffle: the LiDAR rows are the dataset's split -> mask flow row for row (intensity / 10 when fused), the
    virtual rows follow them bin by bin, far -> near."""
    pts = _cloud(2, 50, 80, seed=3)
    pc = (0, -40, -3, 70.4, 40, 1)
    r = osi.front_end(pts, 2, 2, 0.8, later_fusion, shuffle=False, seed=9, pc_range=pc)
    for s in range(2):
        scene = pts[pts[:, 0] == s]
        lidar = scene[scene[:, -1] == 2]
        virt = scene[scene[:, -1] == 1]
        got = r['points'][r['points'][:, 0] == s]
        if later_fusion:
            inr = (lidar[:, 1] >= 0) & (lidar[:, 1] <= np.float32(70.4)) & (np.abs(lidar[:, 2]) <= 40)
            np.testing.assert_array_equal(got, lidar[inr])
            mm = r['points_mm'][r['points_mm'][:, 0] == s]
            assert set(map(bytes, mm)) <= set(map(bytes, virt))
        else:
            nl = int(((lidar[:, 1] >= 0) & (lidar[:, 1] <= np.float32(70.4)) & (np.abs(lidar[:, 2]) <= 40)).sum())
            lid = lidar[(lidar[:, 1] >= 0) & (lidar[:, 1] <= np.float32(70.4)) & (np.abs(lidar[:, 2]) <= 40)].copy()
            lid[:, 4] = lid[:, 4] / np.float32(10)
            np.testing.assert_array_equal(got[:nl], lid)
            xs = got[nl:, 1]
            assert (np.diff(osi.bins(xs, 2)) <= 0).all()                    # far bin first
