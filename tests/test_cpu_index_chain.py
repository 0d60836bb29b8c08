"""The composition rule of chained strided convs (csrc/rulebook.cu header), restated in numpy: every level's output set
computed from the first input set by per-dimension intervals equals oracle/rulebook.py's conv_rulebook applied level by
level, on VirConv-L's down-conv chain, VirConv-T's x-batched eval grid and random geometries (chains of one to four), with
the edge cases the kernel must get right (b = -1 padding rows, coordinates outside the grid, 0 and shape - 1 in every
dimension, empty sets).  A dilated strided conv is a chain of one marked per kernel offset, restated alike."""
import numpy as np
import pytest

from oracle import rulebook as orb

# (ksize, stride, padding) of vir_conv2, vir_conv3, vir_conv4's down convs and conv_out (spconv_backbone.py)
VIRCONV_CHAIN = [((3, 3, 3), (2, 2, 2), (1, 1, 1)), ((3, 3, 3), (2, 2, 2), (1, 1, 1)), ((3, 3, 3), (2, 2, 2), (0, 1, 1)),
                 ((3, 1, 1), (2, 1, 1), (0, 0, 0))]


def in_grid(idx, shape, batch):
    return (idx[:, 0] >= 0) & (idx[:, 0] < batch) & np.all((idx[:, 1:] >= 0) & (idx[:, 1:] < np.asarray(shape)), axis=1)


def per_level(idx, shape, batch, levels):
    """oracle: conv_rulebook level by level over the rows the kernels accept (index_ok)."""
    cur, out = idx[in_grid(idx, shape, batch)], []
    for ks, st, pd, *dl in levels:
        oidx, shape, _, _ = orb.conv_rulebook(cur, shape, ks, st, pd, *dl)
        out.append(oidx)
        cur = oidx
    return out


def composed(idx, shape, batch, levels):
    """numpy restatement of chain_mark_kernel + the bitmap rank: per input row and level the product of per-dimension
    intervals, lo = max(0, ceil((lo + pad - ksize + 1) / stride)), hi = min(oshape - 1, floor((hi + pad) / stride)); the
    output set of a level is the sorted union of its cells (batch-major linear order)."""
    idx = np.asarray(idx, dtype=np.int64)
    ok = in_grid(idx, shape, batch)
    b, lo, hi = idx[ok, 0], idx[ok, 1:].copy(), idx[ok, 1:].copy()
    out = []
    for ks, st, pd in levels:
        oshape = np.array(orb.out_spatial_shape(shape, ks, st, pd, (1,) * len(ks)), dtype=np.int64)
        k, s, p = (np.asarray(v, dtype=np.int64) for v in (ks, st, pd))
        first, last = lo + p - (k - 1), hi + p
        lo = np.where(first <= 0, 0, -(-first // s))
        hi = np.where(last < 0, -1, np.minimum(last // s, oshape - 1))
        live = np.all(lo <= hi, axis=1)
        b, lo, hi = b[live], lo[live], hi[live]
        width = (hi - lo + 1).max(axis=0) if b.size else np.zeros(len(ks), dtype=np.int64)
        cells = []
        for off in np.ndindex(*[int(w) for w in width]):
            c = lo + np.asarray(off, dtype=np.int64)
            m = np.all(c <= hi, axis=1)
            lin = b[m]
            for d in range(len(ks)):
                lin = lin * oshape[d] + c[m, d]
            cells.append(lin)
        out.append(indices(np.unique(np.concatenate(cells)) if cells else np.zeros(0, dtype=np.int64), oshape))
        shape = [int(v) for v in oshape]
    return out


def dilated_mark(idx, shape, batch, ks, st, pd, dl):
    """numpy restatement of conv_mark_kernel on a dilated level 0 (a chain of one): per input row and kernel offset the one
    cell out_cell reaches, o = (c + pad - off * dil) / stride where that divides exactly and 0 <= o < oshape; the output
    set is the sorted union of those cells."""
    idx = np.asarray(idx, dtype=np.int64)
    idx = idx[in_grid(idx, shape, batch)]
    oshape = np.array(orb.out_spatial_shape(shape, ks, st, pd, dl), dtype=np.int64)
    s, p, d = (np.asarray(v, dtype=np.int64) for v in (st, pd, dl))
    cells = []
    for off in np.ndindex(*ks):
        num = idx[:, 1:] + p - np.asarray(off) * d
        o = num // s
        ok = np.all((num >= 0) & (o * s == num) & (o < oshape), axis=1)
        lin = idx[ok, 0]
        for e in range(len(ks)):
            lin = lin * oshape[e] + o[ok, e]
        cells.append(lin)
    return indices(np.unique(np.concatenate(cells)), oshape)


def indices(lin, oshape):
    """batch-major linear cell indices -> [M, 1 + ndim] int32 (b, coordinates)"""
    oidx = np.zeros((lin.size, 1 + len(oshape)), dtype=np.int32)
    rem = lin.copy()
    for d in range(len(oshape) - 1, -1, -1):
        oidx[:, 1 + d] = rem % oshape[d]
        rem //= oshape[d]
    oidx[:, 0] = rem
    return oidx


def random_set(rng, n, shape, batch, edges=True):
    idx = np.stack([rng.integers(0, batch, n)] + [rng.integers(0, s, n) for s in shape], axis=1)
    nd = len(shape)
    if edges:   # 0 and shape - 1 (odd and even extents) in every dimension, both batch ends, and rows the kernels drop
        corners = [[bb] + [c[d] for d in range(nd)] for bb in (0, batch - 1)
                   for c in np.array(np.meshgrid(*[(0, 1, s - 2, s - 1) for s in shape])).reshape(nd, -1).T]
        z = [0] * nd
        bad = ([[-1] + z, [batch] + z, [0, -1] + z[1:]] +
               [[0] + [shape[e] if e == d else 0 for e in range(nd)] for d in range(1, nd)] + [[-1] * (1 + nd)])
        idx = np.concatenate([idx, np.array(corners), np.array(bad)])
    idx = np.unique(idx, axis=0)    # (the 3-D input sets are duplicate-free)
    return idx[rng.permutation(len(idx))].astype(np.int32)


def check(idx, shape, batch, levels):
    want, got = per_level(idx, shape, batch, levels), composed(idx, shape, batch, levels)
    assert len(want) == len(got)
    for lvl, (w, g) in enumerate(zip(want, got)):
        np.testing.assert_array_equal(g, w.reshape(-1, 1 + len(shape)), err_msg=f'level {lvl}')


@pytest.mark.parametrize('shape', [(41, 64, 56), (81, 40, 36), (40, 33, 35), (11, 8, 7)])
@pytest.mark.parametrize('batch', [1, 2, 3])
def test_virconv_chain_random(shape, batch):
    rng = np.random.default_rng(hash((shape, batch)) & 0xFFFF)
    for density in (0.002, 0.03, 0.3):
        n = max(1, int(density * batch * np.prod(shape)))
        check(random_set(rng, n, shape, batch), list(shape), batch, VIRCONV_CHAIN)


def test_xbatched_eval_grid():
    """VirConv-T's ROT_NUM = 3 eval input: three copies side by side along x, [D, H, 4W]."""
    rng = np.random.default_rng(3)
    shape = (41, 40, 4 * 44)
    check(random_set(rng, 3000, shape, 2), list(shape), 2, VIRCONV_CHAIN)


def test_empty_and_single():
    shape = [41, 16, 16]
    check(np.zeros((0, 4), dtype=np.int32), shape, 2, VIRCONV_CHAIN)
    check(np.array([[-1, 0, 0, 0]], dtype=np.int32), shape, 2, VIRCONV_CHAIN)
    for c in ([0, 0, 0], [40, 15, 15], [1, 1, 1], [39, 14, 14]):
        check(np.array([[1] + c], dtype=np.int32), shape, 2, VIRCONV_CHAIN)


def test_random_geometries():
    """Other strided chains of one to four levels with dilation 1: kernel sizes 1-4, strides 1-3, paddings 0-2 (ksize >=
    stride or not)."""
    rng = np.random.default_rng(7)
    for _ in range(40):
        L = int(rng.integers(1, 5))
        levels = [(tuple(int(v) for v in rng.integers(1, 5, 3)), tuple(int(v) for v in rng.integers(1, 4, 3)),
                   tuple(int(v) for v in rng.integers(0, 3, 3))) for _ in range(L)]
        shape = [int(v) for v in rng.integers(20, 60, 3)]
        try:
            sh = shape
            for ks, st, pd in levels:
                sh = orb.out_spatial_shape(sh, ks, st, pd, (1, 1, 1))
                assert min(sh) > 0
        except AssertionError:
            continue
        check(random_set(rng, int(rng.integers(1, 400)), shape, 2), shape, 2, levels)


@pytest.mark.parametrize('nd', [3, 2])
def test_dilated_chain_of_one(nd):
    """A dilated strided conv, a chain of one: dilations 2-3, kernel sizes 1-3, strides 1-3, paddings 0-2, in 3-D and 2-D."""
    rng = np.random.default_rng(11 + nd)
    tried = 0
    for _ in range(40):
        ks, st, pd, dl = (tuple(int(v) for v in rng.integers(lo, hi, nd)) for lo, hi in ((1, 4), (1, 4), (0, 3), (2, 4)))
        shape = [int(v) for v in rng.integers(12, 40, nd)]
        if min(orb.out_spatial_shape(shape, ks, st, pd, dl)) <= 0:
            continue
        idx = random_set(rng, int(rng.integers(1, 400)), shape, 2)
        want = per_level(idx, shape, 2, [(ks, st, pd, dl)])[0]
        np.testing.assert_array_equal(dilated_mark(idx, shape, 2, ks, st, pd, dl), want.reshape(-1, 1 + nd))
        tried += 1
    assert tried >= 20
