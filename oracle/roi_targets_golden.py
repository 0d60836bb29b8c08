"""Record what the reference's OWN `ProposalTargetLayer.forward` and `RoIHeadTemplate.assign_targets` compute, on the
CPU, as tests/golden/roi_targets_ref.npz.  Needs the reference's sources (imported through virconv_b200.reference_env);
the fixture it writes is committed, so the tests need neither.  Three things are patched while the reference runs:

  * `iou3d_nms_utils.boxes_iou3d_gpu` -> the float64 3-D IoU of oracle/iou3d.py, rounded to fp32;
  * `np.random.permutation / rand / randint` and `torch.randint` -> `Draws`, which returns exactly the draws rule 4-5 of
    csrc/roi_targets.cu derives from recorded uniforms (per scene a permutation or a rand call, then one or two randint
    calls; `subsample_rois` is wrapped to mark where a scene starts);
  * `Tensor.cuda` -> the identity.

Case L — VirConv-L's STAGE0 (R = 160, hard sampling on), B = 2, 512 proposals per scene around ~35 GT: ragged GT with
trailing and interior zero rows, a duplicated GT (argmax ties), 32 zero-padded proposals with label 1 (as
proposal_layer emits them), proposals of class 2 that has no GT.
Case S — VirConv-T's STAGE0 (hard sampling off), B = 4, 160 proposals: foreground with only easy background,
foreground-free with hard and easy background, all-zero GT (only easy), only hard background.  (A foreground-only scene
cannot be recorded: the reference's branch for it ends in torch.cat((fg_inds, [])), which raises TypeError.)
Case C — two classes with their own thresholds and a GT class 3 without a threshold entry, B = 2, 300 proposals.
Every overlap is at least MARGIN from every threshold and every non-tied argmax is separated by at least MARGIN, so fp32
against float64 IoU cannot flip a decision; make() checks it.

    python -m oracle.roi_targets_golden REFERENCE_ROOT [OUT_DIR]
"""
from __future__ import annotations

import os
import sys

import numpy as np

MARGIN = 1e-4
SEED = 23
CAR = (3.9, 1.6, 1.56)
SIZES = {1: CAR, 2: (0.8, 0.6, 1.73), 3: (1.76, 0.6, 1.73)}
CFG_L = dict(ROI_PER_IMAGE=160, FG_RATIO=0.5, SAMPLE_ROI_BY_EACH_CLASS=True, CLS_SCORE_TYPE='roi_iou_x',
             CLS_FG_THRESH=[0.75], CLS_BG_THRESH=[0.25], CLS_BG_THRESH_LO=0.1, HARD_BG_RATIO=0.8, REG_FG_THRESH=[0.55],
             ENABLE_HARD_SAMPLING=True, HARD_SAMPLING_THRESH=[0.5], HARD_SAMPLING_RATIO=[0.5])       # VirConv-L.yaml
CFG_S = dict(CFG_L, REG_FG_THRESH=[0.5], ENABLE_HARD_SAMPLING=False)                               # VirConv-T STAGE0
CFG_C = dict(ROI_PER_IMAGE=128, FG_RATIO=0.5, SAMPLE_ROI_BY_EACH_CLASS=True, CLS_SCORE_TYPE='roi_iou_x',
             CLS_FG_THRESH=[0.75, 0.7], CLS_BG_THRESH=[0.25, 0.3], CLS_BG_THRESH_LO=0.1, HARD_BG_RATIO=0.7,
             REG_FG_THRESH=[0.55, 0.45], ENABLE_HARD_SAMPLING=True, HARD_SAMPLING_THRESH=[0.5, 0.35],
             HARD_SAMPLING_RATIO=[0.5, 0.25])
CASES = {'L': CFG_L, 'S': CFG_S, 'C': CFG_C}


def cfg_of(case):
    from virconv_b200.reference_env import EasyDict
    return EasyDict(CASES[case])


def thresholds(cfg):
    t = [cfg['CLS_BG_THRESH_LO']] + list(cfg['REG_FG_THRESH']) + list(cfg['CLS_FG_THRESH']) + list(cfg['CLS_BG_THRESH'])
    if cfg['ENABLE_HARD_SAMPLING']:
        t += list(cfg['HARD_SAMPLING_THRESH'])
    return np.array(t)


def iou64(a, b):
    from oracle import iou3d
    return iou3d.matrix(np.asarray(a, np.float64), np.asarray(b, np.float64), fn=iou3d.iou3d)


def iou_f32(a, b):
    return iou64(a, b).astype(np.float32)


class Draws:
    """The reference's host draws from recorded uniforms (rules 4-5): permutation(n) = the stable argsort of
    u_fg[scene, :n]; rand(R) = u_fg[scene, :R] as float64 (the caller's floor(rand * nf) is then draw(u, nf));
    torch.randint(0, n, (k,)) = draw(u_bg[scene, pos:pos + k], n), pos advancing per call; np.random.randint(0, t) =
    draw(u_hs[i], t), i advancing per call."""

    def __init__(self, u_fg, u_bg, u_hs):
        self.u_fg, self.u_bg, self.u_hs = u_fg, u_bg, u_hs
        self.scene, self.pos, self.hs = -1, 0, 0

    def new_scene(self):
        self.scene += 1
        self.pos = 0

    def permutation(self, n):
        return np.argsort(self.u_fg[self.scene, :n], kind='stable')

    def rand(self, n):
        return self.u_fg[self.scene, :n].astype(np.float64)

    def torch_randint(self, low=0, high=None, size=None, **kw):
        import torch
        from oracle.roi_targets import draw
        assert low == 0
        k = int(size[0])
        idx = draw(self.u_bg[self.scene, self.pos:self.pos + k], int(high))
        self.pos += k
        return torch.from_numpy(np.asarray(idx, np.int64))

    def np_randint(self, low, high=None, size=None):
        from oracle.roi_targets import draw
        assert low == 0 and size is None
        v = int(draw(self.u_hs[self.hs], int(high)))
        self.hs += 1
        return v


def run_reference(cfg, rois, roi_scores, roi_labels, gt, u_fg, u_bg, u_hs):
    """the reference's forward + assign_targets on the CPU with the patches above -> dict of numpy arrays"""
    import types

    import torch
    from pcdet.models.roi_heads.roi_head_template import RoIHeadTemplate
    from pcdet.models.roi_heads.target_assigner import proposal_target_layer as ptl
    draws = Draws(u_fg, u_bg, u_hs)
    saved = (ptl.iou3d_nms_utils.boxes_iou3d_gpu, np.random.permutation, np.random.rand, np.random.randint, torch.randint,
             torch.Tensor.cuda, ptl.ProposalTargetLayer.subsample_rois)
    sub = ptl.ProposalTargetLayer.subsample_rois

    def subsample(self, *a, **k):
        draws.new_scene()
        return sub(self, *a, **k)
    ptl.iou3d_nms_utils.boxes_iou3d_gpu = lambda a, b: torch.from_numpy(iou_f32(a.numpy(), b.numpy()))
    np.random.permutation, np.random.rand, np.random.randint = draws.permutation, draws.rand, draws.np_randint
    torch.randint = draws.torch_randint
    torch.Tensor.cuda = lambda self, *a, **k: self
    ptl.ProposalTargetLayer.subsample_rois = subsample
    try:
        head = types.SimpleNamespace(proposal_target_layers=[ptl.ProposalTargetLayer(roi_sampler_cfg=cfg)])
        batch = {'batch_size': rois.shape[0], 'rois': torch.from_numpy(rois), 'roi_scores': torch.from_numpy(roi_scores),
                 'roi_labels': torch.from_numpy(roi_labels), 'gt_boxes': torch.from_numpy(gt)}
        out = RoIHeadTemplate.assign_targets(head, batch, 0)
    finally:
        (ptl.iou3d_nms_utils.boxes_iou3d_gpu, np.random.permutation, np.random.rand, np.random.randint, torch.randint,
         torch.Tensor.cuda, ptl.ProposalTargetLayer.subsample_rois) = saved
    assert draws.scene == rois.shape[0] - 1
    return {k: v.numpy() for k, v in out.items()}


def heading(rng):
    return np.float32(rng.uniform(-np.pi, np.pi))


def gt_box(rng, cls):
    s = np.array(SIZES[cls], np.float32) * np.float32(rng.uniform(0.85, 1.15))
    return np.array([rng.uniform(5, 65), rng.uniform(-35, 35), rng.uniform(-1.5, 0.0), *s, heading(rng), cls], np.float32)


def near(rng, g, sigma):
    """a proposal around GT row g"""
    b = g[:7].copy()
    b[:2] += rng.normal(0, sigma, 2).astype(np.float32)
    b[2] += np.float32(rng.normal(0, sigma / 3))
    b[3:6] *= rng.uniform(0.8, 1.2, 3).astype(np.float32)
    b[6] = np.float32(b[6] + rng.normal(0, 0.25) + (np.pi if rng.random() < 0.2 else 0.0))
    return b


def far(rng):
    return np.array([rng.uniform(0, 70), rng.uniform(-40, 40), rng.uniform(-1.5, 0.0), *CAR, heading(rng)], np.float32)


def margin_ok(row, cand, thr):
    """row: float64 IoUs of one RoI against the kept GTs, cand: its class's columns"""
    if not len(cand):
        return True
    v = row[cand]
    mx = v.max()
    if np.abs(thr - mx).min() < MARGIN:
        return False
    gap = mx - v[v < mx]
    return not (len(gap) and gap.min() < MARGIN)


def fix_margins(rng, cfg, rois, labels, gt, make, accept=None):
    """resample (with make(i)) every RoI of one scene that breaks the margin or `accept(ov)`"""
    from oracle.roi_targets import trimmed_count
    g = gt[:trimmed_count(gt)]
    cls = g[:, -1].astype(np.int64)
    thr = thresholds(cfg)
    for i in range(len(rois)):
        for _ in range(2000):
            if not rois[i].any():
                break
            row = iou64(rois[i:i + 1, :7], g[:, :7])[0]
            cand = np.nonzero(cls == labels[i])[0]
            ov = row[cand].max() if len(cand) else 0.0
            if margin_ok(row, cand, thr) and (accept is None or accept(ov)):
                break
            rois[i] = make(i)
        else:
            raise RuntimeError('could not place RoI %d' % i)


def case_l(rng):
    cfg = CASES['L']
    B, M, G = 2, 512, 48
    gt = np.zeros((B, G, 8), np.float32)
    rois = np.zeros((B, M, 7), np.float32)
    labels = np.ones((B, M), np.int64)
    for b, n in enumerate((34, 29)):
        rows = [gt_box(rng, 1) for _ in range(n)]
        if b == 0:
            rows.insert(6, rows[5].copy())                                   # duplicated GT: argmax ties
            rows.insert(20, np.zeros(8, np.float32))                          # interior zero row (class 0)
        gt[b, :len(rows)] = np.stack(rows)
        real = [r for r in rows if r.any()]
        n_pad = 32

        def make(i, b=b, real=real):
            if i < 380 or 460 <= i < M - n_pad:
                return near(rng, real[rng.integers(len(real))], rng.choice([0.15, 0.4, 0.9, 2.0]))
            return far(rng)
        for i in range(M - n_pad):
            rois[b, i] = make(i)
        labels[b, 440:460] = 2                                                 # class 2: no GT of it
        fix_margins(rng, cfg, rois[b], labels[b], gt[b], make)
    return rois, labels, gt


def case_s(rng):
    cfg = CASES['S']
    B, M, G = 4, 160, 16
    gt = np.zeros((B, G, 8), np.float32)
    rois = np.zeros((B, M, 7), np.float32)
    labels = np.ones((B, M), np.int64)
    accept = {0: lambda ov: ov >= 0.5 or ov < 0.1, 1: lambda ov: ov < 0.5, 2: None, 3: lambda ov: 0.1 <= ov < 0.5}
    sig = {0: (0.03, 0.08, 8.0), 1: (0.4, 1.5, 6.0), 2: (0.4, 1.5), 3: (0.5, 0.8)}
    for b in range(B):
        if b != 2:
            rows = [gt_box(rng, 1) for _ in range(10 + b)]
            gt[b, :len(rows)] = np.stack(rows)
        real = [r for r in gt[b] if r.any()] or [gt_box(rng, 1)]

        def make(i, b=b, real=real):
            return near(rng, real[rng.integers(len(real))], rng.choice(sig[b]))
        for i in range(M):
            rois[b, i] = make(i)
        fix_margins(rng, cfg, rois[b], labels[b], gt[b], make, accept[b])
    return rois, labels, gt


def case_c(rng):
    cfg = CASES['C']
    B, M, G = 2, 300, 30
    gt = np.zeros((B, G, 8), np.float32)
    rois = np.zeros((B, M, 7), np.float32)
    labels = np.ones((B, M), np.int64)
    for b in range(B):
        rows = [gt_box(rng, c) for c in (1,) * 8 + (2,) * 7 + (3,) * 5]
        rng.shuffle(rows)
        gt[b, :len(rows)] = np.stack(rows)
        real = rows

        def make(i, b=b, real=real):
            g = real[rng.integers(len(real))]
            labels[b, i] = int(g[7]) if rng.random() < 0.9 else int(rng.integers(1, 4))
            return near(rng, g, rng.choice([0.05, 0.15, 0.4, 1.0]))
        for i in range(M):
            rois[b, i] = make(i)
        fix_margins(rng, cfg, rois[b], labels[b], gt[b], make)
    return rois, labels, gt


def make(reference_root, out_dir):
    import virconv_b200.reference_env as renv
    renv.install(reference_root=reference_root)
    rng = np.random.default_rng(SEED)
    res = {}
    for case, build in (('L', case_l), ('S', case_s), ('C', case_c)):
        rois, labels, gt = build(rng)
        B, M = labels.shape
        R = CASES[case]['ROI_PER_IMAGE']
        scores = rng.random((B, M)).astype(np.float32)
        scores[rois.sum(-1) == 0] = 0
        u_fg = rng.random((B, max(M, R)), dtype=np.float32)
        u_bg = rng.random((B, R), dtype=np.float32)
        u_hs = rng.random(len(CASES[case]['REG_FG_THRESH']), dtype=np.float32)
        out = run_reference(cfg_of(case), rois, scores, labels, gt, u_fg, u_bg, u_hs)
        res.update({f'{case}.rois_in': rois, f'{case}.roi_scores_in': scores, f'{case}.roi_labels_in': labels,
                    f'{case}.gt': gt, f'{case}.u_fg': u_fg, f'{case}.u_bg': u_bg, f'{case}.u_hs': u_hs})
        res.update({f'{case}.{k}': v for k, v in out.items()})
        print(case, {k: v.shape for k, v in out.items()}, 'reg_valid', int(out['reg_valid_mask'].sum()),
              'fg-ish', int((out['gt_iou_of_rois'] >= 0.5).sum()))
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'roi_targets_ref.npz')
    np.savez_compressed(path, **res)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    make(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else os.path.join(root, 'tests', 'golden'))
