"""Record what the reference's OWN `AnchorHeadTemplate.get_loss` and `RoIHeadTemplate.get_loss` compute, with the
gradients `torch.autograd.grad` takes of the returned loss with respect to the predictions, as
tests/golden/head_losses_ref.npz.  Needs the reference's sources (imported through virconv_b200.reference_env); the
fixture it writes is committed, so the tests need neither.  The methods run on the CPU on stand-in head objects
(the reference class without its network, with its own build_losses) in float64, with three patches that change dtype
or device only, never the arithmetic:

  * `Tensor.cuda` -> the identity: WeightedSmoothL1Loss.__init__ calls `.cuda()` on its code weights;
  * `common_utils.rotate_points_along_z` -> the same function without the `.float()` on its rotation matrix
    (common_utils.py:53); without it the corner loss fails in float64 with "expected Double but found Float";
  * `roi_head_template.F.binary_cross_entropy` -> casts the target to the input's dtype: get_box_cls_layer_loss passes
    `rcnn_cls_labels.float()`, which fails in float64 with "Found dtype Float but expected Double".  It also passes 0
    for the ignored label -1, which torch's BCE kernels reject (targets outside [0, 1]); those rows are multiplied by
    the valid mask 0 right after, so neither the loss nor a gradient changes.  (-1 comes from CLS_SCORE_TYPE roi_iou;
    the VirConv YAMLs' roi_iou_x makes labels in [0, 1].  The fused loss masks -1 rows as the reference's code states.)

Each case is also recorded once in float32 as the model runs (key prefix `f32.`), with only `Tensor.cuda` and the
BCE target patch (the kernels' range check).

Cases: L — VirConv-L's RPN (1 class, 2 rotations), B = 2, 2000 anchors, labels -1 / 0 / 1 / 2 (2 folds to 1), scene 1
without a positive, NaN targets on codes 0-5, logits beyond +-40; C3 — a 3-class RPN; R1 — RCNN, 3 branches x 1 stage;
R3 — 3 branches x 3 stages, stage 2 without foreground (no corner term, b_loss = 0), soft labels with -1 entries and
logits beyond +-40.  Every discrete decision (direction bin, smooth-L1 branch, min(norm, norm_flip), limit()'s wraps,
the clamps and min / max of compute_iou, the kinks of abs) is at least MARGIN from its switch point, so fp32 cannot flip
it; make() checks it.  T — deliberate ties recorded in float64 only: a foreground row whose source GT has zero length
and width (every corner pair equidistant) and a row whose decoded box equals its target on the x axis (equal edges).

    python -m oracle.head_losses_golden REFERENCE_ROOT [OUT_DIR]
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np

MARGIN = 1e-4
SEED = 31
RPN_L = dict(num_class=1, sets=1, L=1000, B=2)
RPN_C3 = dict(num_class=3, sets=3, L=250, B=2)
RPN_CFG = dict(DIR_OFFSET=0.78539, NUM_DIR_BINS=2, USE_DIRECTION_CLASSIFIER=True,
               LOSS_CONFIG=dict(LOSS_WEIGHTS={'cls_weight': 1.0, 'loc_weight': 2.0, 'dir_weight': 0.2,
                                              'code_weights': [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0]}),
               TARGET_ASSIGNER_CONFIG=dict(BOX_CODER='ResidualCoder'))                          # VirConv-L.yaml
RCNN_CFG = dict(LOSS_CONFIG=dict(CLS_LOSS='BinaryCrossEntropy', REG_LOSS='smooth-l1', CORNER_LOSS_REGULARIZATION=True,
                                 GRID_3D_IOU_LOSS=False,
                                 LOSS_WEIGHTS={'rcnn_cls_weight': 1.0, 'rcnn_reg_weight': 1.0, 'rcnn_corner_weight': 1.0,
                                               'rcnn_iou3d_weight': 1.0,
                                               'code_weights': [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0]}))
RCNN_KEYS = ('rcnn_cls', 'rcnn_reg', 'rois', 'gt_of_rois', 'gt_of_rois_src', 'reg_valid_mask', 'rcnn_cls_labels')
TARGET_KEYS = RCNN_KEYS[2:]


def edict(d):
    from virconv_b200.reference_env import EasyDict
    return EasyDict(d)


def rpn_cfg(num_class):
    from virconv_b200.head_losses import RPNLossConfig
    return RPNLossConfig(edict(RPN_CFG), num_class)


def rcnn_cfg():
    from virconv_b200.head_losses import RCNNLossConfig
    return RCNNLossConfig(edict(RCNN_CFG))


# ---- inputs ---------------------------------------------------------------------------------------------------------
def f32(a):
    return np.asarray(a, np.float32)


def rpn_case(rng, num_class, sets, L, B):
    A = sets * 2
    N = L * A
    anchors = np.zeros((sets, 1, L, 1, 2, 7), np.float32)
    anchors[..., 0] = rng.uniform(0, 70, (1, 1, L, 1, 1))
    anchors[..., 1] = rng.uniform(-40, 40, (1, 1, L, 1, 1))
    anchors[..., 2] = -1.78
    anchors[..., 3:6] = (3.9, 1.6, 1.56)
    anchors[..., 0, 6], anchors[..., 1, 6] = 0.0, 1.57
    labels = rng.choice([-1, 0, 0, 0, 1], size=(B, N)).astype(np.int32)
    if num_class == 1:
        labels[0, rng.choice(N, 20, replace=False)] = 2            # folds to 1
    else:
        pos = labels > 0
        labels[pos] = rng.integers(1, num_class + 1, pos.sum())
    labels[1][labels[1] > 0] = 0                                    # scene 1: no positive
    flat = anchors.transpose(1, 2, 0, 3, 4, 5).reshape(N, 7)       # torch.cat(self.anchors, dim=-3).view(-1, 7)
    tgt = np.zeros((B, N, 7), np.float32)
    pos = labels > 0
    tgt[pos] = f32(rng.normal(0, [0.3, 0.3, 0.3, 0.1, 0.1, 0.1, 1.0], (pos.sum(), 7)))
    cls = f32(rng.normal(0, 2, (B, L, A * num_class)))
    box = f32(rng.normal(0, 0.3, (B, L, A * 7)))
    dirp = f32(rng.normal(0, 1.5, (B, L, A * 2)))
    cls.reshape(B, N, num_class)[0, :8] = f32([45, -45, 60, -41, 50, -50, 42, -70])[:, None]   # saturated logits
    rows = np.nonzero(pos[0])[0][:4]
    tgt[0, rows, rng.integers(0, 6, 4)] = np.nan                     # NaN targets on a few positives
    tgt[0, np.nonzero(labels[0] == 0)[0][:2], 2] = np.nan
    fix_rpn(rng, cls, box, tgt, flat, labels, num_class)
    return dict(cls_preds=cls, box_preds=box, dir_cls_preds=dirp, box_cls_labels=labels, box_reg_targets=tgt,
                anchors=anchors, anchors_flat=flat)


def rpn_margins(cls, box, tgt, flat, num_class):
    """per anchor: True where every decision of R4-R6 is at least MARGIN from its switch point"""
    B = cls.shape[0]
    N = flat.shape[0]
    x = cls.reshape(B, N, num_class).astype(np.float64)
    ok = (np.abs(x) >= MARGIN).all(-1)
    b, t = box.reshape(B, N, 7).astype(np.float64), tgt.astype(np.float64)
    xi, ti = b.copy(), t.copy()
    xi[..., 6] = np.sin(b[..., 6]) * np.cos(t[..., 6])
    ti[..., 6] = np.cos(b[..., 6]) * np.sin(t[..., 6])
    ti = np.where(np.isnan(ti), xi, ti)
    d = np.abs(xi - ti)
    nan = np.isnan(t)
    ok &= ((np.abs(d - 1 / 9) >= MARGIN) & (d >= MARGIN) | nan).all(-1)
    v = (np.nan_to_num(t[..., 6]) + flat[None, :, 6]) - 0.78539
    off = (v - np.floor(v / (2 * np.pi)) * 2 * np.pi) / np.pi       # bin width pi for 2 bins
    ok &= np.abs(off - np.round(off)) >= MARGIN
    return ok


def fix_rpn(rng, cls, box, tgt, flat, labels, num_class):
    B, N = labels.shape
    keep = np.zeros((B, N), bool)
    keep[0, :8] = True                                               # the saturated logits stay
    for _ in range(50):
        bad = ~rpn_margins(cls, box, tgt, flat, num_class) & ~keep
        if not bad.any():
            return
        bb, ii = np.nonzero(bad)
        cv = cls.reshape(B, N, num_class)
        cv[bb, ii] = f32(rng.normal(0, 2, (len(bb), num_class)))
        box.reshape(B, N, 7)[bb, ii] = f32(rng.normal(0, 0.3, (len(bb), 7)))
        t6 = tgt[bb, ii, 6]
        tgt[bb, ii, 6] = np.where(labels[bb, ii] > 0, f32(rng.normal(0, 1.0, len(bb))), t6)
    raise RuntimeError('could not place the RPN inputs away from their switch points')


def canonical(roi, src):
    """gt_of_rois as assign_targets makes it, in float64 (rounded to fp32 by the caller)"""
    g = src[:, :7].astype(np.float64).copy()
    g[:, :3] -= roi[:, :3]
    c, s = np.cos(-roi[:, 6]), np.sin(-roi[:, 6])
    x, y = g[:, 0].copy(), g[:, 1].copy()
    g[:, 0], g[:, 1] = x * c - y * s, x * s + y * c
    h = (src[:, 6] - roi[:, 6]) % (2 * np.pi)
    h = np.where((h > np.pi / 2) & (h < 1.5 * np.pi), (h + np.pi) % (2 * np.pi), h)
    g[:, 6] = np.where(h > np.pi, h - 2 * np.pi, h)
    return g


def target_set(rng, B, R, fg_frac):
    n = B * R
    roi = np.zeros((n, 7))
    roi[:, 0], roi[:, 1], roi[:, 2] = rng.uniform(5, 65, n), rng.uniform(-35, 35, n), rng.uniform(-1.5, 0, n)
    roi[:, 3:6] = np.array([3.9, 1.6, 1.56]) * rng.uniform(0.8, 1.2, (n, 3))
    roi[:, 6] = rng.uniform(-np.pi, np.pi, n)
    roi = f32(roi).astype(np.float64)
    src = np.zeros((n, 8))
    src[:, :7] = roi + rng.normal(0, [0.3, 0.3, 0.1, 0.2, 0.1, 0.1, 0.2], (n, 7))
    src[:, 7] = 1
    src[:, 6] += np.where(rng.random(n) < 0.2, np.pi, 0)             # some GTs opposite: the flipped corners win
    gt = np.zeros((n, 8))
    for _ in range(20):                                              # canonical headings away from limit()'s wraps
        src = f32(src).astype(np.float64)
        gt[:, :7] = canonical(roi, src)
        bad = np.abs(f32(gt[:, 6])) < 1e-3
        if not bad.any():
            break
        src[bad, 6] += 0.01
    gt[:, 7] = 1
    valid = (rng.random(n) < fg_frac).astype(np.int64)
    labels = f32(np.clip(rng.uniform(-0.2, 1.2, n), 0, 1))
    labels[rng.random(n) < 0.1] = -1
    return {'rois': f32(roi).reshape(B, R, 7), 'gt_of_rois': f32(gt).reshape(B, R, 8),
            'gt_of_rois_src': f32(src).reshape(B, R, 8), 'reg_valid_mask': valid.reshape(B, R),
            'rcnn_cls_labels': labels.reshape(B, R)}


def rcnn_margin_rows(t, cfg):
    """per row: True where every decision of C3-C5 is at least MARGIN from its switch point"""
    from oracle import head_losses as o
    n = t['rcnn_reg'].shape[0]
    r = t['rcnn_reg'].astype(np.float64)
    roi = t['rois'].reshape(n, 7).astype(np.float64)
    gt = t['gt_of_rois'].reshape(n, -1)[:, :7].astype(np.float64)
    src = t['gt_of_rois_src'].reshape(n, -1)[:, :7].astype(np.float64)
    x = t['rcnn_cls'].reshape(-1).astype(np.float64)
    ok = np.abs(x) >= MARGIN
    anc = np.zeros((n, 7))
    anc[:, 3:6] = roi[:, 3:6]
    d = np.abs(r - o.encode(gt, anc))
    ok &= ((np.abs(d - 1 / 9) >= MARGIN) & (d >= MARGIN)).all(1)
    a4 = anc.copy()
    a4[:, 6] = roi[:, 6]
    pb = o.decode(r, a4)
    c0, s0 = np.cos(roi[:, 6]), np.sin(roi[:, 6])
    cx, cy = pb[:, 0].copy(), pb[:, 1].copy()
    pb[:, 0], pb[:, 1], pb[:, 2] = cx * c0 - cy * s0 + roi[:, 0], cx * s0 + cy * c0 + roi[:, 1], pb[:, 2] + roi[:, 2]
    gf = src.copy()
    gf[:, 6] += np.pi
    n1 = np.linalg.norm(o.corners(pb) - o.corners(src), axis=-1)
    n2 = np.linalg.norm(o.corners(pb) - o.corners(gf), axis=-1)
    dist = np.minimum(n1, n2)
    ok &= ((np.abs(n1 - n2) >= MARGIN) & (np.abs(dist - 1) >= MARGIN)).all(1)
    pb = o.decode(r, anc)
    for a in range(3):
        hi1, lo1 = pb[:, a] + pb[:, a + 3] * 0.5, pb[:, a] - pb[:, a + 3] * 0.5
        hi2, lo2 = gt[:, a] + gt[:, a + 3] * 0.5, gt[:, a] - gt[:, a + 3] * 0.5
        ov = np.minimum(hi1, hi2) - np.maximum(lo1, lo2)
        ok &= (np.abs(hi1 - hi2) >= MARGIN) & (np.abs(lo1 - lo2) >= MARGIN) & (np.abs(ov) >= MARGIN)
    for h in (pb[:, 6], gt[:, 6]):
        m = h - np.floor(h / (2 * np.pi)) * 2 * np.pi
        ok &= (np.abs(m) >= MARGIN) & (np.abs(m - np.pi) >= MARGIN) & (np.abs(m - 2 * np.pi) >= MARGIN)
    dlt = o.limit(pb[:, 6]) - o.limit(gt[:, 6])
    ok &= (np.abs(np.sin(dlt)) >= MARGIN) & (np.abs(np.cos(pb[:, 6] - gt[:, 6])) >= MARGIN)
    return ok


def rcnn_preds(rng, t, cfg, saturate, keep_rows=()):
    n = t['rois'].shape[0] * t['rois'].shape[1]
    cls = f32(rng.normal(0, 2, (n, 1)))
    if saturate:
        cls[:6, 0] = [45, -45, 41, -60, 80, -41]
    reg = f32(rng.normal(0, [0.15, 0.15, 0.15, 0.08, 0.08, 0.08, 0.2], (n, 7)))
    keep = np.zeros(n, bool)
    keep[:6] = saturate
    keep[list(keep_rows)] = True
    for _ in range(200):
        bad = ~rcnn_margin_rows(dict(t, rcnn_cls=cls, rcnn_reg=reg), cfg) & ~keep
        if not bad.any():
            return cls, reg
        k = int(bad.sum())
        cls[bad, 0] = f32(rng.normal(0, 2, k))
        reg[bad] = f32(rng.normal(0, [0.15, 0.15, 0.15, 0.08, 0.08, 0.08, 0.2], (k, 7)))
    raise RuntimeError('could not place the RCNN predictions away from their switch points')


def rcnn_case(rng, stages, B=2, R=40):
    cfg = rcnn_cfg()
    br = {}
    for i in range(stages):
        t = target_set(rng, B, R, 0.0 if (stages == 3 and i == 2) else 0.45)
        for j, key in enumerate(('targets_dict', 'targets_dict_pi', 'targets_dict_p')):
            cls, reg = rcnn_preds(rng, t, cfg, saturate=(j == 0))
            br[f'{key}{i}'] = dict(t, rcnn_cls=cls, rcnn_reg=reg)
    return br


def tie_case(rng):
    cfg = rcnn_cfg()
    t = target_set(rng, 1, 12, 1.0)
    t['reg_valid_mask'][:] = 1
    t['gt_of_rois_src'][0, 0, 3:5] = 0                            # row 0: zero length and width -> corner ties
    cls, reg = rcnn_preds(rng, t, cfg, saturate=False, keep_rows=(0,))
    reg[1, 0], reg[1, 3] = 0, 0                                   # row 1: decoded x = 0, dx = the RoI's
    t['gt_of_rois'][0, 1, 0] = 0
    t['gt_of_rois'][0, 1, 3] = t['rois'][0, 1, 3]
    return {'targets_dict0': dict(t, rcnn_cls=cls, rcnn_reg=reg)}


# ---- the reference ---------------------------------------------------------------------------------------------------
class _Patched:
    def __init__(self, f64):
        self.f64 = f64

    def __enter__(self):
        import torch
        import torch.nn.functional as F
        from pcdet.models.roi_heads import roi_head_template as rht
        from pcdet.utils import common_utils
        self.saved = (torch.Tensor.cuda, common_utils.rotate_points_along_z, rht.F)
        torch.Tensor.cuda = lambda self, *a, **k: self
        if self.f64:
            def rotate_points_along_z(points, angle):
                cosa, sina = torch.cos(angle), torch.sin(angle)
                zeros, ones = angle.new_zeros(points.shape[0]), angle.new_ones(points.shape[0])
                rot_matrix = torch.stack((cosa, sina, zeros, -sina, cosa, zeros, zeros, zeros, ones), dim=1).view(-1, 3, 3)
                points_rot = torch.matmul(points[:, :, 0:3], rot_matrix)
                return torch.cat((points_rot, points[:, :, 3:]), dim=-1)
            common_utils.rotate_points_along_z = rotate_points_along_z

        class _F(types.ModuleType):
            def __getattr__(self, name):
                return getattr(F, name)

            @staticmethod
            def binary_cross_entropy(input, target, *a, **k):
                return F.binary_cross_entropy(input, target.to(input.dtype).clamp(min=0), *a, **k)
        rht.F = _F('F')
        return self

    def __exit__(self, *exc):
        import torch
        from pcdet.models.roi_heads import roi_head_template as rht
        from pcdet.utils import common_utils
        torch.Tensor.cuda, common_utils.rotate_points_along_z, rht.F = self.saved


def run_rpn(case, num_class, f64):
    import torch
    from pcdet.models.dense_heads.anchor_head_template import AnchorHeadTemplate
    dt = torch.float64 if f64 else torch.float32
    with _Patched(f64):
        head = AnchorHeadTemplate.__new__(AnchorHeadTemplate)
        torch.nn.Module.__init__(head)
        head.model_cfg = edict(RPN_CFG)
        head.num_class = num_class
        head.use_multihead = False
        head.num_anchors_per_location = case['anchors'].shape[0] * 2
        head.build_losses(head.model_cfg.LOSS_CONFIG)
        head.anchors = [torch.from_numpy(a).to(dt) for a in case['anchors']]
        preds = {k: torch.from_numpy(case[k]).to(dt).requires_grad_() for k in ('cls_preds', 'box_preds', 'dir_cls_preds')}
        head.forward_ret_dict = dict(preds, box_cls_labels=torch.from_numpy(case['box_cls_labels'].copy()),
                                     box_reg_targets=torch.from_numpy(case['box_reg_targets']).to(dt))
        loss, tb = head.get_loss()
        grads = torch.autograd.grad(loss, list(preds.values()))
    out = {'loss': np.float64(loss.item()), 'tb': np.array([tb['rpn_loss_cls'], tb['rpn_loss_loc'], tb['rpn_loss_dir'],
                                                            tb['rpn_loss']])}
    out.update({'g_' + k: g.numpy() for k, g in zip(preds, grads)})
    return out


def run_rcnn(case, f64):
    import torch
    from pcdet.models.roi_heads.roi_head_template import RoIHeadTemplate
    from pcdet.utils.box_coder_utils import ResidualCoder
    dt = torch.float64 if f64 else torch.float32
    with _Patched(f64):
        head = RoIHeadTemplate.__new__(RoIHeadTemplate)
        torch.nn.Module.__init__(head)
        head.model_cfg = edict(RCNN_CFG)
        head.box_coder = ResidualCoder(code_size=7)
        head.build_losses(head.model_cfg.LOSS_CONFIG)
        frd, preds = {}, []
        for name, t in case.items():
            d = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in t.items()}
            for k in ('rcnn_cls', 'rcnn_reg', 'rois', 'gt_of_rois', 'gt_of_rois_src'):
                d[k] = d[k].to(dt)
            d['rcnn_cls'].requires_grad_()
            d['rcnn_reg'].requires_grad_()
            preds += [d['rcnn_cls'], d['rcnn_reg']]
            frd[name] = d
        head.forward_ret_dict = frd
        loss, tb = head.get_loss()
        grads = torch.autograd.grad(loss, preds)
    out = {'loss': np.float64(loss.item()), 'tb': np.array([tb['rcnn_loss']])}
    for k, name in enumerate(case):
        out[f'g_cls.{name}'], out[f'g_reg.{name}'] = grads[2 * k].numpy(), grads[2 * k + 1].numpy()
    return out


def branch_order(names):
    """the reference's loop order over the branch names present"""
    from virconv_b200.head_losses import BRANCH_KEYS
    return [(f'{key}{i}', w) for i in range(6) for key, w in BRANCH_KEYS if f'{key}{i}' in names]


def make(reference_root, out_dir):
    import virconv_b200.reference_env as renv
    renv.install(reference_root=reference_root)
    rng = np.random.default_rng(SEED)
    res = {}
    for name, spec in (('L', RPN_L), ('C3', RPN_C3)):
        case = rpn_case(rng, spec['num_class'], spec['sets'], spec['L'], spec['B'])
        assert rpn_margins(case['cls_preds'], case['box_preds'], case['box_reg_targets'], case['anchors_flat'],
                           spec['num_class'])[:, 8:].all()
        res.update({f'{name}.{k}': v for k, v in case.items()})
        for f64, pre in ((True, ''), (False, 'f32.')):
            out = run_rpn(case, spec['num_class'], f64)
            res.update({f'{pre}{name}.{k}': v for k, v in out.items()})
        print(name, 'rpn tb', res[f'{name}.tb'])
    cfg = rcnn_cfg()
    for name, case in (('R1', rcnn_case(rng, 1)), ('R3', rcnn_case(rng, 3)), ('T', tie_case(rng))):
        for bname, t in case.items():
            if name != 'T':
                assert rcnn_margin_rows(t, cfg)[6:].all()
            res.update({f'{name}.{bname}.{k}': v for k, v in t.items()})
        res[f'{name}.branches'] = np.array(list(case))
        for f64, pre in ((True, ''), (False, 'f32.')) if name != 'T' else ((True, ''),):
            out = run_rcnn(case, f64)
            res.update({f'{pre}{name}.{k}': v for k, v in out.items()})
        print(name, 'rcnn tb', res[f'{name}.tb'])
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'head_losses_ref.npz')
    np.savez_compressed(path, **res)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    make(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else os.path.join(root, 'tests', 'golden'))
