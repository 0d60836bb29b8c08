"""Device-drawn StVD layer discard, host side: the numpy oracle of the sampling rule (oracle/stvd_layer.py) and the plans
a paper-mode backbone hands to the executor with discard_rng='device'."""
import numpy as np
import pytest
from scipy import stats

from oracle import stvd_layer as osl

CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG8 = dict(CFG, LAYER_DISCARD_RATE=0.15, MM=True)


def _philox_scalar(ctr, key):
    """Philox4x32-10 with Python integers, one block at a time (an independent restatement of the vectorised oracle)."""
    c, k = list(ctr), list(key)
    m = 0xFFFFFFFF
    for r in range(10):
        if r:
            k = [(k[0] + 0x9E3779B9) & m, (k[1] + 0xBB67AE85) & m]
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k[0], p1 & m, (p0 >> 32) ^ c[3] ^ k[1], p0 & m]
    return c


@pytest.mark.parametrize('ctr,key,want', [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(v) for v in osl.philox4x32_10(ctr, key)) == want
    assert tuple(_philox_scalar(ctr, key)) == want


def test_philox_matches_scalar_restatement():
    rng = np.random.default_rng(1)
    ctr = rng.integers(0, 2 ** 32, size=(200, 4), dtype=np.uint64)
    key = rng.integers(0, 2 ** 32, size=(200, 2), dtype=np.uint64)
    got = osl.philox4x32_10(ctr, key)
    for j in range(200):
        assert [int(v) for v in got[j]] == _philox_scalar([int(v) for v in ctr[j]], [int(v) for v in key[j]])
    # row keys: counter (i, site, 0, 0), key = the seed's two 32-bit halves (two's complement for a negative seed)
    seed = -0x123456789abcdef
    u = osl.row_keys(64, 3, seed)
    s = seed & (2 ** 64 - 1)
    assert [int(v) for v in u] == [_philox_scalar([i, 3, 0, 0], [s & 0xFFFFFFFF, s >> 32])[0] for i in range(64)]


@pytest.mark.parametrize('rate', [0.1, 0.15, 0.5])
def test_keep_count_is_python_float64_arithmetic(rate):
    """k = int(n * (1 - rate)) for every n <= 300 000, as float64 products truncated (what the device and the executor
    compute); a float32 rate would give other counts (n = 10 at 0.1: 8 instead of 9)."""
    n = np.arange(300001)
    dev = np.trunc(n.astype(np.float64) * (1.0 - rate)).astype(np.int64)
    assert np.array_equal(dev, np.array([osl.keep_count(int(v), rate) for v in n]))
    if rate == 0.1:
        assert int(10 * (1 - np.float64(np.float32(rate)))) == 8 and osl.keep_count(10, rate) == 9


@pytest.mark.parametrize('n', [0, 1, 2, 31, 33, 1000, 4097])
@pytest.mark.parametrize('rate', [0.1, 0.5, 1.0])
def test_selection_is_smallest_keys_in_row_order(n, rate):
    for seed in (0, 7, -3):
        u = osl.row_keys(n, 1, seed)
        keep = osl.keep_rows(n, rate, 1, seed)
        k = int(n * (1 - rate))
        assert keep.shape == (k,) and np.all(np.diff(keep) > 0)
        assert np.array_equal(keep, np.sort(np.lexsort((np.arange(n), u))[:k]))
        if k and k < n:       # every kept key is at most every dropped key
            dropped = np.setdiff1d(np.arange(n), keep)
            assert u[keep].max() <= u[dropped].min()


def test_tie_rule_takes_lowest_rows_first():
    keys = np.array([5, 1, 5, 5, 0, 5, 1, 5], dtype=np.uint32)
    assert osl.keep_rows(8, 0.5, 0, 0, keys=keys).tolist() == [0, 1, 4, 6]       # (0,4) (1,1) (1,6) (5,0)
    assert osl.keep_rows(8, 0.25, 0, 0, keys=keys).tolist() == [0, 1, 2, 3, 4, 6]
    rng = np.random.default_rng(3)
    keys = rng.integers(0, 4, size=5000).astype(np.uint32)                      # heavy duplicates
    keep = osl.keep_rows(5000, 0.37, 0, 0, keys=keys)
    assert np.array_equal(keep, np.sort(np.lexsort((np.arange(5000), keys))[:int(5000 * 0.63)]))


def test_inclusion_is_uniform_over_seeds():
    """Each row is kept with probability k / n: chi-square of the per-row inclusion counts over 4000 seeds."""
    n, rate, S = 60, 0.15, 4000
    k = int(n * (1 - rate))
    counts = np.zeros(n)
    for seed in range(S):
        counts[osl.keep_rows(n, rate, 2, seed * 0x9E3779B97F4A7C15 % 2 ** 63)] += 1
    p = k / n
    chi2 = float(((counts - S * p) ** 2 / (S * p * (1 - p))).sum())
    assert stats.chi2.sf(chi2, n - 1) > 1e-4, chi2
    # and the pairwise structure of a k-subset: the number kept is always exactly k
    assert counts.sum() == S * k


def _ops(plan):
    return plan.finalize()[0]


def test_device_discard_plan_rows():
    """paper + 'device', training: a DISCARD op (index stream, float64 rate in two int32 halves, site 0-2) right after the
    concat of vir_conv1..3, before the next block's strided conv; it is what publish() marks.  Eval mode, the 'numpy' draw
    and the default mode keep the default plan row for row."""
    import torch
    from virconv_b200 import executor
    from virconv_b200.backbone import VirConvL8x
    default = _ops(VirConvL8x(CFG, 8, [1408, 1600, 80])._plan())
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], discard_mode='paper', discard_rng='device')
    oi = _ops(m._plan())
    assert oi.shape[0] == default.shape[0] + 3
    disc = [i for i in range(oi.shape[0]) if oi[i, 0] == executor.OP_DISCARD]
    assert len(disc) == 3
    for site, i in enumerate(disc):
        r = oi[i]
        assert r[1] == 1 and r[4] == site and r[22] == 1
        assert oi[i - 1, 0] == executor.OP_CAT and oi[i - 1, 4] == r[18]       # gathers the concat just built
        assert oi[i + 1, 0] == executor.OP_CONV_RB and oi[i + 1, 2] == r[3]    # the next strided conv reads its rows
        assert np.array([r[6], r[7]], dtype=np.int32).view(np.float64)[0] == 0.1
    assert np.array_equal(np.delete(oi, disc, axis=0)[:, :2], default[:, :2])
    assert [n for n, _, _ in m._plan().published] == ['x_conv1', 'x_conv2', 'x_conv3', 'x_conv4', 'out']
    # publish() marks the discard, not the concat that feeds it
    assert all(oi[i - 1, 22] == 0 for i in disc)
    m.eval()
    assert np.array_equal(_ops(m._plan()), default)
    m.train()
    assert m._plan() is m._plan_stvd_cache and m._plan_cache is not None           # both cached
    numpy_draw = VirConvL8x(CFG, 8, [1408, 1600, 80], discard_mode='paper')
    assert np.array_equal(_ops(numpy_draw._plan()), default)
    assert not numpy_draw._use_plan(torch.zeros((4, 8)))
    # index-set groups: each published tensor's rulebooks are those of its own rows
    plan = m._plan()
    groups = {name: plan.iset_group[s] for name, _, s in plan.published}
    assert groups == {'x_conv1': 1, 'x_conv2': 2, 'x_conv3': 3, 'x_conv4': 3, 'out': 3}


def test_virconv8x_mm_device_discard_plan():
    from virconv_b200 import executor
    from virconv_b200.backbone import VirConv8x
    m = VirConv8x(CFG8, 8, [1408, 1600, 80], discard_mode='paper', discard_rng='device')
    oi = _ops(m._plan_mm(True))
    disc = [i for i in range(oi.shape[0]) if oi[i, 0] == executor.OP_DISCARD]
    assert disc[0] == 0 and [oi[i, 4] for i in disc] == [0, 1, 2, 3]
    assert oi[0, 2] == 0 and oi[0, 18] == 0                                    # site 0: the input voxels
    # no parameter gradient flows into the input: the first conv after the input discard computes no input gradient
    first_cbr = next(r for r in oi if r[0] == executor.OP_CBR)
    assert first_cbr[2] == oi[0, 19] and first_cbr[21] == 0
    assert np.array_equal(_ops(m._plan_mm()), _ops(VirConv8x(CFG8, 8, [1408, 1600, 80])._plan_mm()))
    assert not any(r[0] == executor.OP_DISCARD for r in _ops(m._plan_lidar()))


def test_discard_plan_without_seed_is_rejected(lib_built):
    """vc_exec_forward (no seed) refuses a plan with a layer discard before any CUDA call."""
    from virconv_b200 import _lib
    from virconv_b200.backbone import VirConvL8x
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], discard_mode='paper', discard_rng='device')
    oi, of, lf, _, _ = m._plan().finalize()
    lib = _lib.load()
    state = np.zeros(lib.vc_exec_state_bytes(), dtype=np.uint8)
    rc = lib.vc_exec_forward(oi.ctypes.data, of.ctypes.data, oi.shape[0], None, None, lf.shape[0], None, 8, None, 1,
                             _lib.host_i32([41, 1600, 1408]), 2, None, 1, 0, 1, None, 0, None, None, state.ctypes.data, state.size,
                             None, None, 1, None, None, None, None)
    assert rc == -1 and b'needs a seed' in lib.vc_last_error()
