"""The gather-form input gradient of the many-to-one 2-D tables (oracle/gather2d.py, run by the deterministic mode's
csrc/gather2d.cu) is the scatter-form gradient of oracle/rulebook.py's rule 3, up to the summation order."""
import numpy as np
import pytest

from oracle import gather2d as og
from oracle import rulebook as orb


def _case(coords, shape, cin, cout, seed):
    rng = np.random.default_rng(seed)
    nbr = orb.subm_rulebook(coords, shape, 3)
    w = rng.standard_normal((cout, 9, cin))
    dout = rng.standard_normal((coords.shape[0], cout))
    rep = og.representatives(coords, shape)
    want = og.scatter_dgrad(dout, w, nbr)
    got = og.gather_dgrad(dout, w, nbr, rep)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-300)), rep


def _coords(rng, n, batch, shape):
    return np.stack([rng.integers(0, batch, n)] + [rng.integers(0, s, n) for s in shape], 1).astype(np.int32)


def test_heavy_duplication_stride8_image():
    """~20 k rows on ~3 k pixels, like the stride-8 image of a VirConv-L batch"""
    rng = np.random.default_rng(8)
    c = _coords(rng, 20000, 2, [48, 36])
    err, rep = _case(c, [48, 36], 32, 64, 1)
    assert 2500 < np.unique(rep).size < 3500
    assert err < 1e-12


def test_no_duplicates():
    rng = np.random.default_rng(3)
    c = np.unique(_coords(rng, 3000, 2, [60, 70]), axis=0)
    rng.shuffle(c)
    err, rep = _case(c, [60, 70], 16, 16, 2)
    assert np.array_equal(rep, np.arange(c.shape[0]))
    assert err < 1e-12


def test_single_row():
    err, rep = _case(np.array([[0, 4, 5]], np.int32), [9, 9], 8, 16, 3)
    assert err < 1e-12 and rep.tolist() == [0]


@pytest.mark.parametrize('seed', [0, 1])
def test_two_batch_elements_share_pixels(seed):
    """(b, u, v) is the key: the same (u, v) in two batch elements are different pixels"""
    rng = np.random.default_rng(seed)
    uv = rng.integers(0, 12, (400, 2))
    c = np.concatenate([np.concatenate([np.zeros((400, 1)), uv], 1), np.concatenate([np.ones((400, 1)), uv], 1)]).astype(np.int32)
    c = c[rng.permutation(c.shape[0])]
    err, rep = _case(c, [12, 12], 16, 32, 4 + seed)
    assert np.all(c[rep, 0] == c[:, 0])
    assert err < 1e-12
