"""Record what the reference's OWN `TEDMHead.obtain_conf_preds` (ted_head.py:425-442, with its `gen_sample_grid` and
`bilinear_interpolate_torch_gridsample`, :110-156) computes, with the part-map gradient `torch.autograd.grad` takes for a
seeded upstream gradient, as tests/golden/part_pool_ref.npz.  Needs the reference's sources (imported through
virconv_b200.reference_env); the fixture it writes is committed, so the tests need neither.  The method runs on the CPU
on a stand-in head (the reference class without its network, with the `gen_grid_fn` its __init__ builds, :382-383).

Each case is recorded twice: in float32 as the model runs (key prefix `f32.`), and in float64 with the one patch
oracle/head_losses_golden.py documents, `common_utils.rotate_points_along_z` without the `.float()` on its rotation
matrix (common_utils.py:53), which would otherwise fail on float64 points.

Cases (maps of about 40 x 36 instead of KITTI's 200 x 176; the full size is checked against oracle/part_pool.py on the
GPU):
  A — B = 1, N = 160, VirConv-T's GRID_OFFSETS / FEATMAP_STRIDE: headings 0, +-pi/2, pi and random; RoIs inside the map,
      straddling each of its four borders and fully outside; zero-size boxes; 24 copies of one box (every tap collides);
      20 all-zero padding rows;
  B — B = 2, N = 50, random RoIs, scene 1 ending in zero rows;
  C — B = 1, N = 1;
  D — B = 2, N = 50 on a 16 x 32 map with FEATMAP_STRIDE 0.25: zero-size and heading-0 boxes on dyadic centres and
      sizes, so that samples fall exactly on integer and half-integer pixel coordinates, in both precisions; some at
      the borders.
Every sample that is not exact in both precisions stays at least MARGIN px from an integer coordinate, so floor()
cannot flip between the reference, the oracle and the kernel; make() asserts it.

    python -m oracle.part_pool_golden REFERENCE_ROOT [OUT_DIR]
"""
from __future__ import annotations

import os
import sys

import numpy as np

MARGIN = 1e-3
SEED = 47
S = 7
KITTI = dict(offsets=(0.0, 40.0), stride=0.4, H=40, W=36)      # VirConv-T.yaml PART: GRID_OFFSETS, FEATMAP_STRIDE
DYADIC = dict(offsets=(0.0, 2.0), stride=0.25, H=16, W=32)


def f32(a):
    return np.asarray(a, np.float32)


def geom_of(z, case):
    """(S, offsets, scale, featmap_stride) of a recorded case"""
    g = z[f'{case}.geom']
    return int(g[0]), (float(g[1]), float(g[2])), 1 / float(g[3]), float(g[3])


def sample_ok(rois, geo):
    """per RoI: True where every sample is either exact (on a half-integer grid, equal in fp32 and float64) or at least
    MARGIN from an integer coordinate in x and in y"""
    from oracle import part_pool as o
    scale = 1 / geo['stride']
    ix, iy = o.positions(rois, S, geo['offsets'], scale, geo['H'], geo['W'])
    ix32, iy32 = o.positions(f32(rois), S, geo['offsets'], scale, geo['H'], geo['W'], dtype=np.float32)
    ok = np.ones(ix.shape, bool)
    for a, a32 in ((ix, ix32), (iy, iy32)):
        exact = (a * 2 == np.round(a * 2)) & (a32.astype(np.float64) == a)
        ok &= exact | (np.abs(a - np.round(a)) >= MARGIN)
    return ok.all(-1)


def random_rois(rng, n, geo, lo=-0.1, hi=1.1):
    """boxes with centres over [lo, hi] of the map (pixel fractions), car-like sizes, random headings"""
    sc = 1 / geo['stride']
    r = np.zeros((n, 7))
    r[:, 0] = rng.uniform(lo, hi, n) * geo['W'] / sc - geo['offsets'][0]
    r[:, 1] = rng.uniform(lo, hi, n) * geo['H'] / sc - geo['offsets'][1]
    r[:, 2] = rng.uniform(-1.5, 0.0, n)
    r[:, 3] = rng.uniform(1.5, 4.5, n) * geo['stride'] / 0.4
    r[:, 4] = rng.uniform(1.2, 2.0, n) * geo['stride'] / 0.4
    r[:, 5] = 1.5
    r[:, 6] = rng.uniform(-np.pi, np.pi, n)
    return r


def at_pixel(geo, X, Y):
    """the centre (x, y) whose sample lands at pixel coordinate (X, Y) of the map"""
    sc = 1 / geo['stride']
    return X / sc - geo['offsets'][0], Y / sc - geo['offsets'][1]


def fix(rng, rois, geo, keep):
    """redraw the centres of rows (not in `keep`) whose samples come too close to an integer coordinate"""
    for _ in range(200):
        bad = ~sample_ok(rois, geo) & ~keep
        if not bad.any():
            return rois
        k = int(bad.sum())
        rois[bad, 0] += f32(rng.uniform(-0.05, 0.05, k))
        rois[bad, 1] += f32(rng.uniform(-0.05, 0.05, k))
    raise RuntimeError('could not place the RoIs away from integer sample coordinates')


def case_a(rng):
    geo = KITTI
    H, W = geo['H'], geo['W']
    r = random_rois(rng, 160, geo)
    cx, cy = at_pixel(geo, W / 2, H / 2)
    r[0:4, 0], r[0:4, 1] = cx + 0.13, cy + 0.07
    r[0:4, 6] = [0.0, np.pi / 2, -np.pi / 2, np.pi]
    for k, (X, Y) in enumerate(((0.5, H / 2), (W - 0.7, H / 2), (W / 2, 0.6), (W / 2, H - 0.4))):   # four borders
        r[4 + k, 0], r[4 + k, 1] = at_pixel(geo, X + 0.011, Y + 0.013)
        r[4 + k, 6] = 0.3 * k
    r[8, 0], r[8, 1] = at_pixel(geo, -20.0, H / 2)                    # fully outside
    r[9, 0], r[9, 1] = at_pixel(geo, W / 2, H + 25.0)
    r[10:12, 3:5] = 0                                                 # zero-size boxes
    r[12:36] = r[36]                                                  # 24 copies of one box
    r[140:] = 0                                                       # proposal padding
    r = f32(r).astype(np.float64)
    keep = np.zeros(160, bool)
    keep[140:] = True
    r = fix(rng, r, geo, keep)
    r[12:37] = r[36]
    return f32(r)[None], geo


def case_b(rng):
    geo = KITTI
    r = random_rois(rng, 100, geo).reshape(2, 50, 7)
    r[0, :3, 6] = [0.0, np.pi, -np.pi / 2]
    r[1, 45:] = 0
    keep = np.zeros((2, 50), bool)
    keep[1, 45:] = True
    r = fix(rng, f32(r).astype(np.float64).reshape(100, 7), geo, keep.reshape(-1)).reshape(2, 50, 7)
    return f32(r), geo


def case_c(rng):
    geo = KITTI
    r = fix(rng, f32(random_rois(rng, 1, geo, 0.3, 0.7)).astype(np.float64), geo, np.zeros(1, bool))
    return f32(r)[None], geo


def case_d(rng):
    """dyadic: centres on multiples of 1/8 m (1/2 px at scale 4), sizes multiples of 1/4 m"""
    geo = DYADIC
    H, W = geo['H'], geo['W']
    r = np.zeros((2, 50, 7))
    r[..., 0] = rng.integers(0, 2 * W + 1, (2, 50)) / 2 / 4 - geo['offsets'][0]
    r[..., 1] = rng.integers(0, 2 * H + 1, (2, 50)) / 2 / 4 - geo['offsets'][1]
    r[..., 2] = -1.0
    r[:, :20, 3:5] = 0                                                # zero-size: 49 exact samples each
    r[:, 20:, 3] = rng.integers(1, 9, (2, 30)) / 4
    r[:, 20:, 4] = rng.integers(1, 9, (2, 30)) / 4
    r[..., 5] = 1.5
    r[0, 0, 0:2] = at_pixel(geo, 0.0, 0.0)                            # corners of the map
    r[0, 1, 0:2] = at_pixel(geo, W, H)
    r[0, 2, 0:2] = at_pixel(geo, W - 0.5, H - 0.5)
    r[1, 0, 0:2] = at_pixel(geo, 0.5, H / 2)
    ok = sample_ok(r.reshape(100, 7), geo).reshape(2, 50)
    for b, n in zip(*np.nonzero(~ok)):                                # boxes whose inner samples come near an integer
        for _ in range(100):
            r[b, n, 3] = rng.integers(1, 9) / 4
            r[b, n, 4] = rng.integers(1, 9) / 4
            r[b, n, 3] += 1 / 64
            if sample_ok(r[b, n][None], geo).all():
                break
        else:
            raise RuntimeError('could not size a dyadic box')
    return f32(r), geo


def run(parts, rois, g, geo, f64):
    """the reference's obtain_conf_preds and its part-map gradient"""
    from functools import partial

    import torch
    from pcdet.models.roi_heads import ted_head
    from pcdet.utils import common_utils
    dt = torch.float64 if f64 else torch.float32
    saved = common_utils.rotate_points_along_z
    if f64:
        def rotate_points_along_z(points, angle):
            cosa, sina = torch.cos(angle), torch.sin(angle)
            zeros, ones = angle.new_zeros(points.shape[0]), angle.new_ones(points.shape[0])
            rot_matrix = torch.stack((cosa, sina, zeros, -sina, cosa, zeros, zeros, zeros, ones), dim=1).view(-1, 3, 3)
            points_rot = torch.matmul(points[:, :, 0:3], rot_matrix)
            return torch.cat((points_rot, points[:, :, 3:]), dim=-1)
        common_utils.rotate_points_along_z = rotate_points_along_z
    try:
        head = ted_head.TEDMHead.__new__(ted_head.TEDMHead)
        torch.nn.Module.__init__(head)
        head.grid_offsets = list(geo['offsets'])
        head.featmap_stride = geo['stride']
        head.gen_grid_fn = partial(ted_head.gen_sample_grid, grid_offsets=head.grid_offsets,
                                   spatial_scale=1 / head.featmap_stride)
        p = torch.from_numpy(parts).to(dt).requires_grad_()
        out = ted_head.TEDMHead.obtain_conf_preds(head, p, torch.from_numpy(rois).to(dt))
        (dp,) = torch.autograd.grad(out, [p], torch.from_numpy(g).to(dt).view(-1, 1))
    finally:
        common_utils.rotate_points_along_z = saved
    return out.detach().numpy(), dp.numpy()


def make(reference_root, out_dir):
    import virconv_b200.reference_env as renv
    renv.install(reference_root=reference_root)
    rng = np.random.default_rng(SEED)
    res = {}
    for name, fn in (('A', case_a), ('B', case_b), ('C', case_c), ('D', case_d)):
        rois, geo = fn(rng)
        B, N = rois.shape[:2]
        assert sample_ok(rois.reshape(B * N, 7).astype(np.float64), geo).all(), name
        parts = f32(rng.integers(-16, 17, (B, S * S, geo['H'], geo['W'])) / 8)     # dyadic values: exact in both dtypes
        g = f32(rng.integers(-64, 65, B * N) / 16)
        res.update({f'{name}.parts': parts, f'{name}.rois': rois, f'{name}.g': g,
                    f'{name}.geom': np.array([S, geo['offsets'][0], geo['offsets'][1], geo['stride']])})
        for f64, pre in ((True, ''), (False, 'f32.')):
            out, dp = run(parts, rois, g, geo, f64)
            res[f'{pre}{name}.out'], res[f'{pre}{name}.dparts'] = out, dp
        print(name, rois.shape, 'out range', res[f'{name}.out'].min(), res[f'{name}.out'].max())
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'part_pool_ref.npz')
    np.savez_compressed(path, **res)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    make(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else os.path.join(root, 'tests', 'golden'))
