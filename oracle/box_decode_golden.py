"""Record what the reference's OWN box decoding and stage transforms compute, with the box_preds gradients
`torch.autograd.grad` takes for a seeded upstream gradient, as tests/golden/box_decode_ref.npz:
`AnchorHeadTemplate.generate_predicted_boxes` (anchor_head_template.py:335-382), `RoIHeadTemplate.generate_predicted_boxes`
(roi_head_template.py:294-324) and `TEDMHead.roi_x_trans / roi_score_trans / pred_x_trans` (ted_head.py:675-746, over
X_TRANS of X_transform.py).  Needs the reference's sources (imported through virconv_b200.reference_env); the fixture it
writes is committed, so the tests need neither.  The methods run on the CPU on stand-in heads (`box_coder`, `model_cfg`,
`anchors`, `use_multihead`, `x_trans_train`: the attributes the methods read, built from the reference's classes).

Each case is recorded in float32 as the model runs (key prefix `f32.`) and in float64, with the one patch
oracle/head_losses_golden.py documents: `common_utils.rotate_points_along_z` without the `.float()` on its rotation matrix
(common_utils.py:53), which would otherwise fail on float64 points.

Cases:
  RPN (VirConv-T's anchor generator: 200 x 176 locations x 2 rotations, DIR_OFFSET 0.78539, DIR_LIMIT_OFFSET 0, 2 bins):
    A1 — B = 1, the full anchor set (no gradient recorded);  A2 — B = 2, a masked subset (the locations
    get_anchor_mask keeps around two points);  A3 — B = 1, a smaller masked subset without a direction classifier.
    Residuals and direction logits are dyadic and mostly repeat (so the fixture compresses), with tied logits; headings 0, +-pi/2, pi and values within a
    few ulp of a limit_period bin edge are planted on heading-0 anchors.
    `{case}.amb` marks the anchors whose bin differs between torch's CPU division by the period (the reference here) and
    the CUDA multiplication by its float32 reciprocal (the kernel's rule): there the kernel's heading may differ by one
    period.
  RCNN: R1 — B = 1, N = 1;  R50 — B = 2, N = 50 with 9-column RoIs;  R160 — B = 2, N = 160 with headings 0, +-pi/2, pi
    and zero-size RoIs.
  X_TRANS: boxes [2, 20, 9]; transform_param of scene 0 is VirConv-T.yaml's (rotation (0.3, 0.3, 0), flip (0, 1, 1),
    scale (0.98, 1.02, 1)), scene 1 another set; R = 1, 2, 3 (the first R stages) with rot_num_id 0..2 for each of the
    three methods, so the `while rot_num_id >= R` clamp and roi_x_trans's stage -1 at rot_num_id 0 are covered.  The
    key `X.{method}.{R}.{stage}` holds the result for the clamped stage: make() asserts that every rot_num_id beyond R
    gives exactly the result of the stage it clamps to, and stores it once.

Arrays of two or more axes are stored column-major (save / load), which keeps the fixture small.

    python -m oracle.box_decode_golden REFERENCE_ROOT [OUT_DIR]
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np

SEED = 53
DIR_OFFSET, DIR_LIMIT_OFFSET, NUM_DIR_BINS = 0.78539, 0.0, 2
XT_VIRCONV_T = [[0.3, 0.0, 0.98], [0.3, 1.0, 1.02], [0.0, 1.0, 1.0]]   # per stage: rotation, flip, scale
XT_OTHER = [[-0.2, 1.0, 1.05], [0.45, 0.0, 0.97], [-0.1, 1.0, 1.0]]
XT_METHODS = ('roi_x_trans', 'roi_score_trans', 'pred_x_trans')


COLUMN_MAJOR = '@cm'    # key suffix of an array stored with its last axis first: box columns compress far better apart


def f32(a):
    return np.asarray(a, np.float32)


def save(path, res):
    """np.savez_compressed with every array of two or more axes stored column-major (key + COLUMN_MAJOR)"""
    out = {}
    for k, v in res.items():
        v = np.asarray(v)
        if v.ndim >= 2:
            out[k + COLUMN_MAJOR] = np.ascontiguousarray(np.moveaxis(v, -1, 0))
        else:
            out[k] = v
    np.savez_compressed(path, **out)


def load(path):
    """the fixture save() wrote, as {key: array} in the recorded layout"""
    z = np.load(path)
    res = {}
    for k in z.files:
        if k.endswith(COLUMN_MAJOR):
            res[k[:-len(COLUMN_MAJOR)]] = np.ascontiguousarray(np.moveaxis(z[k], 0, -1))
        else:
            res[k] = z[k]
    return res


def dyadic(rng, shape, p_zero, lo=-8, hi=8, den=8):
    v = rng.integers(lo, hi + 1, shape) / den
    v[rng.random(shape) < p_zero] = 0
    return f32(v)


def edge_headings():
    """float32 headings h (on a heading-0 anchor: h = t6 exactly) for which (h - DIR_OFFSET) / period lies on or within a
    few ulp of an integer, plus 0, +-pi/2, pi"""
    off, p = np.float32(DIR_OFFSET), np.float32(2 * np.pi / NUM_DIR_BINS)
    out = [0.0, np.pi / 2, -np.pi / 2, np.pi]
    for k in (-1, 0, 1):
        h = np.float32(k * p + off)
        for _ in range(4):
            h = np.nextafter(h, np.float32(-10))
        for _ in range(9):
            out.append(h)
            h = np.nextafter(h, np.float32(10))
    return f32(out)


def ambiguous(h32):
    """bins that differ between the division and the reciprocal multiplication (float32)"""
    from oracle import box_decode as o
    val = f32(h32) - np.float32(DIR_OFFSET)
    p = 2 * np.pi / NUM_DIR_BINS
    a = np.floor(o.bin_quotient(val, p, DIR_LIMIT_OFFSET, np.float32, div=True))
    b = np.floor(o.bin_quotient(val, p, DIR_LIMIT_OFFSET, np.float32, div=False))
    return a != b


def virconv_t_anchors():
    """VirConv-T's anchors from the reference's own AnchorGenerator: [200, 176, 1, 2, 7] -> [70400, 7] float32"""
    import torch
    from pcdet.models.dense_heads.target_assigner.anchor_generator import AnchorGenerator
    cfg = [{'class_name': 'Car', 'anchor_sizes': [[3.9, 1.6, 1.56]], 'anchor_rotations': [0, 1.57],
            'anchor_bottom_heights': [-1.78], 'align_center': False, 'feature_map_stride': 8}]
    gen = AnchorGenerator(anchor_range=[0, -40, -3, 70.4, 40, 1], anchor_generator_config=cfg)
    saved = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        anchors, _ = gen.generate_anchors([np.array([176, 200])])
    finally:
        torch.Tensor.cuda = saved
    return anchors[0].numpy().reshape(-1, 7), anchors[0].shape


def _patched(f64):
    from pcdet.utils import common_utils

    from oracle import box_decode as o

    class Patch:
        def __enter__(self):
            self.saved = common_utils.rotate_points_along_z
            if f64:
                common_utils.rotate_points_along_z = o.torch_rotate_points_along_z

        def __exit__(self, *a):
            common_utils.rotate_points_along_z = self.saved
    return Patch()


def run_rpn(box, anchors, dirs, g, f64):
    import torch
    from pcdet.models.dense_heads.anchor_head_template import AnchorHeadTemplate
    from pcdet.utils import box_coder_utils
    dt = torch.float64 if f64 else torch.float32
    B, A = box.shape[:2]
    head = types.SimpleNamespace(
        anchors=[torch.from_numpy(anchors).to(dt).view(1, A // 2, 1, 2, 7)], use_multihead=False,
        box_coder=box_coder_utils.ResidualCoder(),
        model_cfg=types.SimpleNamespace(DIR_OFFSET=DIR_OFFSET, DIR_LIMIT_OFFSET=DIR_LIMIT_OFFSET,
                                        NUM_DIR_BINS=NUM_DIR_BINS))
    bp = torch.from_numpy(box).to(dt).requires_grad_()
    cls = torch.zeros(B, A, 1, dtype=dt)
    d = torch.from_numpy(dirs).to(dt) if dirs is not None else None
    _, out = AnchorHeadTemplate.generate_predicted_boxes(head, B, cls, bp.view(B, A // 2, 14),
                                                         d.view(B, A // 2, 4) if d is not None else None)
    if g is None:
        return out.detach().numpy(), None
    (db,) = torch.autograd.grad(out, [bp], torch.from_numpy(g).to(dt))
    return out.detach().numpy(), db.numpy()


def run_rcnn(box, rois, g, f64):
    import torch
    from pcdet.models.roi_heads.roi_head_template import RoIHeadTemplate
    from pcdet.utils import box_coder_utils
    dt = torch.float64 if f64 else torch.float32
    B, N = rois.shape[:2]
    head = types.SimpleNamespace(box_coder=box_coder_utils.ResidualCoder())
    bp = torch.from_numpy(box).to(dt).requires_grad_()
    with _patched(f64):
        _, out = RoIHeadTemplate.generate_predicted_boxes(head, B, torch.from_numpy(rois).to(dt),
                                                          torch.zeros(B * N, 1, dtype=dt), bp)
    (db,) = torch.autograd.grad(out, [bp], torch.from_numpy(g).to(dt))
    return out.detach().numpy(), db.numpy()


def clamp(i, R):
    """the stage the reference's `while rot_num_id >= R: rot_num_id -= 1` leaves"""
    return min(i, R - 1)


def rpn_anchors(z, case):
    """the anchors [A, 7] of an RPN case: the rows `{case}.sel` of VirConv-T's full set (all of them without it)"""
    return z['anchors'][z[f'{case}.sel']] if f'{case}.sel' in z else z['anchors']


def run_xtrans(method, boxes, tparam, i, f64):
    import torch
    from pcdet.datasets.augmentor.X_transform import X_TRANS
    from pcdet.models.roi_heads.ted_head import TEDMHead
    dt = torch.float64 if f64 else torch.float32
    head = types.SimpleNamespace(x_trans_train=X_TRANS())
    with _patched(f64):
        out = getattr(TEDMHead, method)(head, torch.from_numpy(boxes).to(dt), i, torch.from_numpy(tparam).to(dt))
    return out.numpy()


def rpn_case(rng, anchors, mask, B, with_dir, p_zero, plant):
    sel = np.nonzero(mask)[0]
    A = len(sel)
    anc = anchors[sel]
    box = dyadic(rng, (B, A, 7), p_zero)
    box[..., 3:6] = dyadic(rng, (B, A, 3), p_zero, -4, 4)
    if plant:
        h = edge_headings()
        zero_rot = np.nonzero(anc[:, 6] == 0)[0]
        for b in range(B):
            at = rng.choice(zero_rot, len(h), replace=False)
            box[b, at, 6] = h
    dirs = None
    if with_dir:
        dirs = dyadic(rng, (B, A, NUM_DIR_BINS), 0.5, -1, 1, 4)
        dirs[:, :max(8, A // 50), 1] = dirs[:, :max(8, A // 50), 0]                 # tied logits
    g = dyadic(rng, (B, A, 7), 0.5, -16, 16, 16)
    return anc, box, dirs, g


def rois_of(rng, B, N, ld):
    r = np.zeros((B, N, ld))
    r[..., 0] = rng.uniform(0, 70, (B, N))
    r[..., 1] = rng.uniform(-40, 40, (B, N))
    r[..., 2] = rng.uniform(-2, 0, (B, N))
    r[..., 3] = rng.uniform(3, 4.5, (B, N))
    r[..., 4] = rng.uniform(1.4, 1.9, (B, N))
    r[..., 5] = rng.uniform(1.3, 1.7, (B, N))
    r[..., 6] = rng.uniform(-np.pi, np.pi, (B, N))
    if ld > 7:
        r[..., 7:] = rng.uniform(-1, 1, (B, N, ld - 7))
    return r


def make(reference_root, out_dir):
    import virconv_b200.reference_env as renv
    renv.install(reference_root=reference_root)
    rng = np.random.default_rng(SEED)
    res = {}
    anchors, shape = virconv_t_anchors()
    assert shape == (1, 200, 176, 1, 2, 7), shape
    A_full = anchors.shape[0]
    loc = np.zeros((200, 176), bool)
    for cy, cx in ((40, 30), (170, 150)):
        loc[cy - 5:cy + 5, cx - 5:cx + 5] = True
    mask2 = np.repeat(loc.reshape(-1), 2)
    loc3 = np.zeros((200, 176), bool)
    loc3[0:10, 0:10] = True
    mask3 = np.repeat(loc3.reshape(-1), 2)
    res['anchors'] = anchors
    for name, mask, B, with_dir, p_zero in (('A1', np.ones(A_full, bool), 1, True, 0.97), ('A2', mask2, 2, True, 0.5),
                                            ('A3', mask3, 1, False, 0.3)):
        anc, box, dirs, g = rpn_case(rng, anchors, mask, B, with_dir, p_zero, plant=with_dir)
        if name == 'A1':
            g = None                    # the full set's gradient is checked against the oracle on the GPU
        res[f'{name}.box'] = box
        if not mask.all():
            res[f'{name}.sel'] = np.nonzero(mask)[0].astype(np.int32)
        if g is not None:
            res[f'{name}.g'] = g
        if dirs is not None:
            res[f'{name}.dir'] = dirs
            res[f'{name}.amb'] = ambiguous(box[..., 6] + anc[None, :, 6])
        for f64, pre in ((True, ''), (False, 'f32.')):
            out, db = run_rpn(box, anc, dirs, g, f64)
            res[f'{pre}{name}.out'] = out
            if db is not None:
                res[f'{pre}{name}.dbox'] = db
        print(name, box.shape, 'ambiguous', int(res.get(f'{name}.amb', np.zeros(1)).sum()))
    for name, B, N, ld in (('R1', 1, 1, 7), ('R50', 2, 50, 9), ('R160', 2, 160, 7)):
        rois = rois_of(rng, B, N, ld)
        if name == 'R160':
            rois[0, :4, 6] = [0.0, np.pi / 2, -np.pi / 2, np.pi]
            rois[1, :3, 3:6] = 0                                                      # zero-size RoIs
            rois[1, 3, 3:5] = 0
        if name == 'R50':
            rois[1, -2:, 3:6] = 0
        rois = f32(rois)
        box = f32(rng.normal(0, 0.3, (B * N, 7)))
        g = f32(rng.integers(-64, 65, (B, N, 7)) / 16)
        res.update({f'{name}.rois': rois, f'{name}.box': box, f'{name}.g': g})
        for f64, pre in ((True, ''), (False, 'f32.')):
            out, db = run_rcnn(box, rois, g, f64)
            res[f'{pre}{name}.out'], res[f'{pre}{name}.dbox'] = out, db
    boxes = rois_of(rng, 2, 20, 9)
    boxes[0, :4, 6] = [0.0, np.pi / 2, -np.pi / 2, np.pi]
    boxes[1, :2, 0:3] = 0
    boxes = f32(boxes)
    tparam = f32([XT_VIRCONV_T, XT_OTHER])
    res['X.boxes'], res['X.tparam'] = boxes, tparam
    for R in (1, 2, 3):
        tp = np.ascontiguousarray(tparam[:, :R])
        for m in XT_METHODS:
            for i in range(3):
                for f64, pre in ((True, ''), (False, 'f32.')):
                    key = f'{pre}X.{m}.{R}.{clamp(i, R)}'
                    out = run_xtrans(m, boxes, tp, i, f64)
                    if key in res:          # rot_num_id beyond R: the reference clamps it to a stage already recorded
                        assert np.array_equal(out, res[key]), key
                    else:
                        res[key] = out
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'box_decode_ref.npz')
    save(path, res)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    make(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else os.path.join(root, 'tests', 'golden'))
