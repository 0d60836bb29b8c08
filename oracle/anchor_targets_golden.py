"""Record what the reference's OWN `AnchorHeadSingle.get_anchor_mask` and `AxisAlignedTargetAssigner.assign_targets`
compute, on the CPU, as tests/golden/anchor_targets_ref.npz.  Needs the reference's sources (imported through
virconv_b200.reference_env, with `Tensor.cuda` made the identity: both call `.cuda()` on host-built tensors); the fixture
it writes is committed, so the tests need neither.

Case L — VirConv-L's anchor config (one Car set, two rotations, stride 8: the full 200 x 176 map), masked by points of
scenes.make_points_batch (a subsample, so that the mask has holes) plus points at the low x / y edges and just below them
(both wraps of rule 0), B = 2: scene 0 has ragged GT with zero padding, an interior zero row, a class-0 row (wraps to
the last class name), a duplicated box (argmax ties) and tiny boxes inside several anchors (tied column maxima, several
forced anchors per GT); scene 1's GT rows are all zero (row 0 stays: gt_ious +0.0).
Case T — three anchor sets (Car / Pedestrian / Cyclist, KITTI sizes and thresholds, stride 32, a seeded mask): the
interleaved output order and per-set thresholds; scene 1 has no cyclist (gt_ious -0.0 on that set's anchors).
Headings are drawn at least 1e-5 away from the pi/4 swap and the limit_period wrap.  Anchors are stored as the
generator's 1-D shift vectors (oracle.anchor_targets.anchors_from_shifts rebuilds them).

    python -m oracle.anchor_targets_golden REFERENCE_ROOT [OUT_DIR]
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np

PCR = np.array([0.0, -40.0, -3.0, 70.4, 40.0, 1.0], np.float32)
GRID = np.array([1408, 1600, 80], np.int64)
CLASS_NAMES_L = ['Car']
CLASS_NAMES_T = ['Car', 'Pedestrian', 'Cyclist']
CAR = dict(class_name='Car', anchor_sizes=[[3.9, 1.6, 1.56]], anchor_rotations=[0, 1.57], anchor_bottom_heights=[-1.78],
           align_center=False, feature_map_stride=8, matched_threshold=0.6, unmatched_threshold=0.45)   # VirConv-L.yaml
SETS_T = [dict(CAR, feature_map_stride=32),
          dict(class_name='Pedestrian', anchor_sizes=[[0.8, 0.6, 1.73]], anchor_rotations=[0, 1.57],
               anchor_bottom_heights=[-0.6], align_center=False, feature_map_stride=32, matched_threshold=0.5,
               unmatched_threshold=0.35),
          dict(class_name='Cyclist', anchor_sizes=[[1.76, 0.6, 1.73]], anchor_rotations=[0, 1.57],
               anchor_bottom_heights=[-0.6], align_center=False, feature_map_stride=32, matched_threshold=0.5,
               unmatched_threshold=0.35)]
SIZES = {1: (3.9, 1.6, 1.56), 2: (0.8, 0.6, 1.73), 3: (1.76, 0.6, 1.73)}
FEATURE_SHAPE_L = (2, 384, 200, 176)
M_GT = 40
SEED = 11


def model_cfg(sets):
    from virconv_b200.reference_env import EasyDict
    return EasyDict(ANCHOR_GENERATOR_CONFIG=[EasyDict(s) for s in sets],
                    TARGET_ASSIGNER_CONFIG=EasyDict(NAME='AxisAlignedTargetAssigner', POS_FRACTION=-1.0, SAMPLE_SIZE=512,
                                                    NORM_BY_NUM_EXAMPLES=False, MATCH_HEIGHT=False,
                                                    BOX_CODER='ResidualCoder'))


def heading(rng):
    """uniform in (-pi, pi), at least 1e-5 from the swap (|limit_period| = pi/4) and the wrap (h = pi/2 + k pi)"""
    while True:
        h = np.float32(rng.uniform(-np.pi, np.pi))
        r = float(h) - np.floor(float(h) / np.pi + 0.5) * np.pi
        if abs(abs(r) - np.pi / 4) > 1e-5 and abs(abs(r) - np.pi / 2) > 1e-5:
            return h


def box(rng, centre, cls, scale=(0.85, 1.15)):
    s = np.array(SIZES[cls], np.float32) * np.float32(rng.uniform(*scale))
    z = rng.uniform(-1.5, 0.0)
    return np.array([centre[0], centre[1], z, s[0], s[1], s[2], heading(rng), cls], np.float32)


def points_l(rng):
    from virconv_b200 import scenes
    pb = scenes.make_points_batch([0, 1], n_lidar=2048, n_virtual=4000, training=True)
    pts = pb.points[rng.choice(len(pb.points), 90, replace=False)][:, :3]
    edge = np.array([[0, 1.0, 3.0], [0, 35.0, -39.5], [1, 3.5, -38.0],       # coarse cell 0 -> the fine windows wrap
                     [1, -5.0, 10.0], [0, 50.0, -45.0]], np.float32)       # just below the range -> the coarse index wraps
    return np.ascontiguousarray(np.concatenate([pts, edge]).astype(np.float32))


def gt_l(rng, anchors):
    """scene 0: ragged, with the special rows; scene 1: all zero"""
    loc = anchors.reshape(-1, 7)[:, :2]
    rows = []
    for k in range(22):
        rows.append(box(rng, loc[rng.integers(len(loc))] + rng.normal(0, 0.6, 2).astype(np.float32), 1))
    rows.insert(4, rows[3].copy())                                           # duplicated box
    for k in range(4):                                                        # tiny boxes inside several anchors
        c = loc[rng.integers(len(loc))]
        rows.append(np.array([c[0] + 0.05, c[1] - 0.03, -1.0, 0.12, 0.1, 0.5, 0.0, 1], np.float32))
    rows.insert(10, np.zeros(8, np.float32))                                 # interior zero row
    cls0 = box(rng, loc[rng.integers(len(loc))], 1)
    cls0[7] = 0
    rows.insert(15, cls0)                                                     # class 0 -> class_names[-1]
    gt = np.zeros((2, M_GT, 8), np.float32)
    gt[0, :len(rows)] = np.stack(rows)
    return gt


def gt_t(rng, anchors):
    loc = anchors.reshape(-1, 7)[:, :2]
    gt = np.zeros((2, M_GT, 8), np.float32)
    for b, counts in enumerate(((10, 8, 6), (9, 7, 0))):
        rows = [box(rng, loc[rng.integers(len(loc))] + rng.normal(0, 0.5, 2).astype(np.float32), c)
                for c, n in zip((1, 2, 3), counts) for _ in range(n)]
        rng.shuffle(rows)
        if b == 0:
            rows[5][7] = 0                                                    # wraps to 'Cyclist'
        gt[b, :len(rows)] = np.stack(rows)
    return gt


def make(reference_root, out_dir):
    import torch
    import virconv_b200.reference_env as renv
    from oracle import anchor_targets as o
    renv.install(reference_root=reference_root)
    from pcdet.models.dense_heads.anchor_head_single import AnchorHeadSingle
    from pcdet.models.dense_heads.anchor_head_template import AnchorHeadTemplate
    from pcdet.models.dense_heads.target_assigner.axis_aligned_target_assigner import AxisAlignedTargetAssigner
    from pcdet.utils.box_coder_utils import ResidualCoder

    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        rng = np.random.default_rng(SEED)
        res = {}
        # case L
        anchors, _ = AnchorHeadTemplate.generate_anchors([CAR], GRID, PCR, 7)
        pts = points_l(rng)
        head = types.SimpleNamespace(voxel_size=(PCR[3] - PCR[0]) / GRID[0], range=PCR)
        mask = AnchorHeadSingle.get_anchor_mask(head, {'points': torch.from_numpy(pts)}, FEATURE_SHAPE_L)
        masked = [a[:, mask, ...] for a in anchors]
        gt = gt_l(rng, masked[0].numpy())
        assigner = AxisAlignedTargetAssigner(model_cfg([CAR]), CLASS_NAMES_L, ResidualCoder(), GRID, PCR)
        out = assigner.assign_targets(masked, torch.from_numpy(gt))
        res.update({'L.points': pts, 'L.mask': mask.numpy(), 'L.gt': gt,
                    'L.x_shifts0': anchors[0][0, 0, :, 0, 0, 0].numpy(), 'L.y_shifts0': anchors[0][0, :, 0, 0, 0, 1].numpy()})
        res.update({'L.' + k: v.numpy() for k, v in out.items()})
        # case T
        anchors, _ = AnchorHeadTemplate.generate_anchors(SETS_T, GRID, PCR, 7)
        mask_t = torch.from_numpy(rng.random(anchors[0].shape[1:3]) < 0.7)
        masked = [a[:, mask_t, ...] for a in anchors]
        gt = gt_t(rng, masked[0].numpy())
        assigner = AxisAlignedTargetAssigner(model_cfg(SETS_T), CLASS_NAMES_T, ResidualCoder(), GRID, PCR)
        out = assigner.assign_targets(masked, torch.from_numpy(gt))
        res.update({'T.mask': mask_t.numpy(), 'T.gt': gt})
        for s, a in enumerate(anchors):
            res[f'T.x_shifts{s}'] = a[0, 0, :, 0, 0, 0].numpy()
            res[f'T.y_shifts{s}'] = a[0, :, 0, 0, 0, 1].numpy()
        res.update({'T.' + k: v.numpy() for k, v in out.items()})
    finally:
        torch.Tensor.cuda = cuda
    # the shift vectors rebuild the generator's anchors exactly
    for case, sets in (('L', [CAR]), ('T', SETS_T)):
        for s, cfg in enumerate(sets):
            a = o.anchors_from_shifts(res[f'{case}.x_shifts{s}'], res[f'{case}.y_shifts{s}'], cfg['anchor_bottom_heights'],
                                      cfg['anchor_sizes'], cfg['anchor_rotations'])
            m = res[f'{case}.mask']
            assert a[:, m].shape[1] == int(m.sum())
    lab = res['L.box_cls_labels']
    print('L: mask %.2f of %s, N = %d, positives %d, ignored %d' % (res['L.mask'].mean(), res['L.mask'].shape, lab.shape[1],
                                                                   (lab > 0).sum(), (lab < 0).sum()))
    lab = res['T.box_cls_labels']
    print('T: N = %d, labels %s' % (lab.shape[1], {int(v): int((lab == v).sum()) for v in np.unique(lab)}))
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'anchor_targets_ref.npz')
    np.savez_compressed(path, **res)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    make(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else os.path.join(root, 'tests', 'golden'))
