"""Detection losses, forward + backward: the reference's get_loss control flow restated over torch on the GPU (its
.item() reads and boolean-mask indexing, anchor_head_template.py:178-333, roi_head_template.py:161-291, bbloss.py,
loss_utils.py) against the fused calls of virconv_b200.head_losses, on the same seeded inputs in one process.  Prints the
device name and power limit, the synchronised host time per call (median of the timed window), and the largest
differences of the losses and gradients between the two arms.

    python profiles/microbench_head_losses.py [--iters 50]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))

from oracle import head_losses_golden as g            # noqa: E402
from virconv_b200 import head_losses as hl            # noqa: E402


# ---- the reference's control flow over torch ------------------------------------------------------------------------
def ref_rpn(cls_preds, box_preds, dir_preds, labels, tgt, anchors, cfg):
    B = cls_preds.shape[0]
    labels = labels.clone()
    cared, positives, negatives = labels >= 0, labels > 0, labels == 0
    cls_weights = (negatives * 1.0 + 1.0 * positives).float()
    reg_weights = positives.float()
    if cfg.num_class == 1:
        labels[positives] = 1
    pos_norm = positives.sum(1, keepdim=True).float()
    reg_weights /= torch.clamp(pos_norm, min=1.0)
    cls_weights /= torch.clamp(pos_norm, min=1.0)
    ct = labels * cared.type_as(labels)
    one_hot = torch.zeros(*list(ct.shape), cfg.num_class + 1, dtype=cls_preds.dtype, device=ct.device)
    one_hot.scatter_(-1, ct.unsqueeze(-1).long(), 1.0)
    x = cls_preds.view(B, -1, cfg.num_class)
    t = one_hot[..., 1:]
    p = torch.sigmoid(x)
    fw = (t * cfg.alpha + (1 - t) * (1 - cfg.alpha)) * torch.pow(t * (1.0 - p) + (1.0 - t) * p, cfg.gamma)
    bce = torch.clamp(x, min=0) - x * t + torch.log1p(torch.exp(-torch.abs(x)))
    cls_loss = (fw * bce * cls_weights.unsqueeze(-1)).sum() / B * cfg.cls_weight
    tb = {'rpn_loss_cls': cls_loss.item()}
    bp = box_preds.view(B, -1, 7)
    b1 = torch.cat([bp[..., :6], torch.sin(bp[..., 6:7]) * torch.cos(tgt[..., 6:7])], -1)
    b2 = torch.cat([tgt[..., :6], torch.cos(bp[..., 6:7]) * torch.sin(tgt[..., 6:7])], -1)
    b2 = torch.where(torch.isnan(b2), b1, b2)
    d = (b1 - b2) * torch.tensor(cfg.code_weights, device=bp.device).view(1, 1, -1)
    n = torch.abs(d)
    loc = torch.where(n < cfg.beta, 0.5 * n ** 2 / cfg.beta, n - 0.5 * cfg.beta) * reg_weights.unsqueeze(-1)
    loc_loss = loc.sum() / B * cfg.loc_weight
    tb['rpn_loss_loc'] = loc_loss.item()
    rot = tgt[..., 6] + anchors.view(1, -1, 7).repeat(B, 1, 1)[..., 6]
    v = rot - cfg.dir_offset
    off = v - torch.floor(v / (2 * np.pi)) * (2 * np.pi)
    dt = torch.clamp(torch.floor(off / (2 * np.pi / cfg.num_dir_bins)).long(), min=0, max=cfg.num_dir_bins - 1)
    logits = dir_preds.view(B, -1, cfg.num_dir_bins)
    w = positives.type_as(logits)
    w /= torch.clamp(w.sum(-1, keepdim=True), min=1.0)
    dir_loss = (F.cross_entropy(logits.permute(0, 2, 1), dt, reduction='none') * w).sum() / B * cfg.dir_weight
    tb['rpn_loss_dir'] = dir_loss.item()
    loss = cls_loss + loc_loss + dir_loss
    tb['rpn_loss'] = loss.item()
    return loss, tb


def _encode(g_, a):
    a = a.clone()
    g_ = g_.clone()
    a[:, 3:6] = torch.clamp_min(a[:, 3:6], 1e-5)
    g_[:, 3:6] = torch.clamp_min(g_[:, 3:6], 1e-5)
    diag = torch.sqrt(a[:, 3] ** 2 + a[:, 4] ** 2)
    return torch.stack([(g_[:, 0] - a[:, 0]) / diag, (g_[:, 1] - a[:, 1]) / diag, (g_[:, 2] - a[:, 2]) / a[:, 5],
                        torch.log(g_[:, 3] / a[:, 3]), torch.log(g_[:, 4] / a[:, 4]), torch.log(g_[:, 5] / a[:, 5]),
                        g_[:, 6] - a[:, 6]], -1)


def _decode(t, a):
    diag = torch.sqrt(a[:, 3] ** 2 + a[:, 4] ** 2)
    return torch.stack([t[:, 0] * diag + a[:, 0], t[:, 1] * diag + a[:, 1], t[:, 2] * a[:, 5] + a[:, 2],
                        torch.exp(t[:, 3]) * a[:, 3], torch.exp(t[:, 4]) * a[:, 4], torch.exp(t[:, 5]) * a[:, 5],
                        t[:, 6] + a[:, 6]], -1)


def _rot(points, angle):
    c, s = torch.cos(angle), torch.sin(angle)
    z, o = angle.new_zeros(points.shape[0]), angle.new_ones(points.shape[0])
    m = torch.stack((c, s, z, -s, c, z, z, z, o), dim=1).view(-1, 3, 3).float()
    return torch.cat((torch.matmul(points[:, :, 0:3], m), points[:, :, 3:]), dim=-1)


def _corners(b):
    tpl = b.new_tensor([[1, 1, -1], [1, -1, -1], [-1, -1, -1], [-1, 1, -1], [1, 1, 1], [1, -1, 1], [-1, -1, 1],
                        [-1, 1, 1]]) / 2
    c = b[:, None, 3:6].repeat(1, 8, 1) * tpl[None]
    return _rot(c.view(-1, 8, 3), b[:, 6]).view(-1, 8, 3) + b[:, None, 0:3]


def _iou1(x, w, y, l):
    hi1, lo1, hi2, lo2 = x + w * 0.5, x - w * 0.5, y + l * 0.5, y - l * 0.5
    return (torch.min(hi1, hi2) - torch.max(lo1, lo2)).clamp_min(0.) / (torch.max(hi1, hi2) - torch.min(lo1, lo2)).clamp_min(0.)


def _limit(a):
    a = a % (2 * np.pi)
    a[a > np.pi] = a[a > np.pi] - 2 * np.pi
    a[a < -np.pi] = a[a < -np.pi] + 2 * np.pi
    return a


def ref_rcnn_branch(t, cfg):
    lab = t['rcnn_cls_labels'].view(-1)
    bl = F.binary_cross_entropy(torch.sigmoid(t['rcnn_cls'].view(-1)), lab.float(), reduction='none')
    vm = (lab >= 0).float()
    cls = (bl * vm).sum() / torch.clamp(vm.sum(), min=1.0) * cfg.cls_weight
    cls.item()
    valid = t['reg_valid_mask'].view(-1)
    gct = t['gt_of_rois'][..., 0:7].reshape(-1, 7)
    src = t['gt_of_rois_src'][..., 0:7].reshape(-1, 7)
    reg_p = t['rcnn_reg']
    rois = t['rois'].reshape(-1, 7)
    n = gct.shape[0]
    fg_mask = valid > 0
    fg_sum = fg_mask.long().sum().item()
    ra = rois.clone().detach()
    ra[:, 0:3] = 0
    ra[:, 6] = 0
    tg = _encode(gct, ra)
    d = (reg_p - torch.where(torch.isnan(tg), reg_p, tg)) * torch.tensor(cfg.code_weights, device=reg_p.device)
    nn_ = torch.abs(d)
    rl = torch.where(nn_ < cfg.beta, 0.5 * nn_ ** 2 / cfg.beta, nn_ - 0.5 * cfg.beta)
    reg = (rl * fg_mask.unsqueeze(-1).float()).sum() / max(fg_sum, 1) * cfg.reg_weight
    reg.item()
    if cfg.corner and fg_sum > 0:
        fr, fb = reg_p[fg_mask], rois[fg_mask]
        ba = fb.clone().detach()
        ba[:, 0:3] = 0
        pb = _decode(fr, ba)
        pb = _rot(pb.unsqueeze(1), fb[:, 6]).squeeze(1)
        pb = torch.cat([pb[:, 0:3] + fb[:, 0:3], pb[:, 3:]], -1)
        gs = src[fg_mask]
        gf = gs.clone()
        gf[:, 6] += np.pi
        pc = _corners(pb)
        dist = torch.min(torch.norm(pc - _corners(gs), dim=2), torch.norm(pc - _corners(gf), dim=2))
        cl = torch.where(dist < 1.0, 0.5 * dist ** 2, dist - 0.5).mean(1).mean() * cfg.corner_weight
        reg = reg + cl
        cl.item()
    pb = _decode(reg_p, ra)
    if len(gct[fg_mask]) == 0:
        bb = 0
    else:
        p, q = pb[fg_mask], gct[fg_mask]
        iou = _iou1(p[:, 0], p[:, 3], q[:, 0], q[:, 3]) * _iou1(p[:, 1], p[:, 4], q[:, 1], q[:, 4]) * \
            _iou1(p[:, 2], p[:, 5], q[:, 2], q[:, 5]) * (1 - torch.abs(torch.sin(_limit(p[:, 6]) - _limit(q[:, 6]))))
        af = 1.25 * (1.0 - torch.abs(torch.cos(p[:, -1] - q[:, -1])))
        bb = ((1 - iou + af + torch.pow(q[:, 0:3] - p[:, 0:3], 2).sum(-1)) * 1.5).sum() / (fg_mask.sum() + 1)
    return cls, reg + bb


def ref_rcnn(branches, cfg):
    loss = 0
    for t, w in branches:
        c, r = ref_rcnn_branch(t, cfg)
        loss = loss + w * c + w * r
    return loss, {'rcnn_loss': loss.item()}


# ---- timing -----------------------------------------------------------------------------------------------------------
def timed(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts)), 1e3 * float(np.min(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    args = ap.parse_args()
    from test_gpu_head_losses import full_rpn, virconv_t_branches
    name = torch.cuda.get_device_name()
    q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    print(f'device: {name}, power limit: {q.stdout.strip() or "unknown"}')
    cfg = g.rpn_cfg(1)
    for L in (21800, 35200):
        cls, box, dirp, labels, tgt, anchors = (torch.from_numpy(a).cuda() for a in full_rpn(7, L=L))
        preds = [t.clone().requires_grad_() for t in (cls, box, dirp)]

        def fused():
            loss, stats = hl.rpn_loss(*preds, labels, tgt, anchors, cfg)
            return torch.autograd.grad(loss, preds), stats

        def ref():
            loss, tb = ref_rpn(*preds, labels, tgt, anchors, cfg)
            return torch.autograd.grad(loss, preds), torch.tensor(list(tb.values()))
        (gf, sf), (gr, sr) = fused(), ref()
        dl = float((sf.cpu().double() - sr.double()).abs().max() / sr.abs().max())
        dg = max(float((a - b).abs().max() / b.abs().max()) for a, b in zip(gf, gr))
        tr, tf = timed(ref, args.iters), timed(fused, args.iters)
        print(f'RPN 2 x {2 * L}: reference {tr[0]:.3f} ms (min {tr[1]:.3f}), fused {tf[0]:.3f} ms (min {tf[1]:.3f}); '
              f'max rel diff loss {dl:.2e}, grads {dg:.2e}')
    rcfg = g.rcnn_cfg()
    for label, nb in (('VirConv-L 3 branches', 3), ('VirConv-T 9 branches', 9)):
        branches, _ = virconv_t_branches(8)
        # labels in [0, 1] as roi_iou_x makes them: torch's BCE kernels reject the -1 of other score types
        branches = [({k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in t.items()}, w)
                    for t, w in branches[:nb]]
        for t, _ in branches:
            t['rcnn_cls_labels'] = t['rcnn_cls_labels'].clamp(min=0)
        preds = []
        for t, _ in branches:
            t['rcnn_cls'].requires_grad_()
            t['rcnn_reg'].requires_grad_()
            preds += [t['rcnn_cls'], t['rcnn_reg']]

        def fused():
            loss, stats = hl.rcnn_loss(branches, rcfg)
            return torch.autograd.grad(loss, preds), stats[-1:]

        def ref():
            loss, tb = ref_rcnn(branches, rcfg)
            return torch.autograd.grad(loss, preds), torch.tensor([tb['rcnn_loss']])
        (gf, sf), (gr, sr) = fused(), ref()
        dl = float((sf.cpu().double() - sr.double()).abs().max() / sr.abs().max())
        dg = max(float((a - b).abs().max() / max(float(b.abs().max()), 1e-30)) for a, b in zip(gf, gr))
        tr, tf = timed(ref, args.iters), timed(fused, args.iters)
        print(f'RCNN {label} of 2 x 160: reference {tr[0]:.3f} ms (min {tr[1]:.3f}), fused {tf[0]:.3f} ms '
              f'(min {tf[1]:.3f}); max rel diff loss {dl:.2e}, grads {dg:.2e}')


if __name__ == '__main__':
    main()
