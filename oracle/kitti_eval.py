"""numpy restatement of the KITTI evaluation (kitti_object_eval_python/eval.py: get_official_eval_result), written from
its semantics for the CPU tests of virconv_b200.kitti_eval, plus the seeded synthetic annotations the tests, the golden
generator and the microbenchmark evaluate.

The geometry follows the rules csrc/kitti_eval_geom.cuh states (E1-E4); the matching is compute_statistics_jit's greedy
rule, run for one frame over a vector of lanes (class x difficulty x overlap setting [x threshold]) at once.

    overlaps(gt_annos, dt_annos, metric)       per frame [n_dt, n_gt] float64 blocks
    evaluate(gt_annos, dt_annos, classes, min_overlaps, compute_aos)
                                               {'overlaps', 'thresholds', 'pr', 'precision', 'recall', 'orientation'}
    synthetic_annos(seed, n_frames, ...)       (gt_annos, dt_annos)
"""
from __future__ import annotations

import math

import numpy as np

CLASS_NAMES = ('car', 'pedestrian', 'cyclist', 'van', 'person_sitting', 'truck')
MIN_HEIGHT = (40, 25, 25)
MAX_OCCLUSION = (0, 1, 2)
MAX_TRUNCATION = (0.15, 0.3, 0.5)
N_SAMPLE_PTS = 41
F32 = np.float32


# ---------------------------------------------------------------------------------------------------------------- geometry
def _corners(b):
    """E1: b = (x, y, dx, dy, angle) float32 -> 8 float32 corner coordinates.  cos / sin rounded from float64, as the
    kernel does (numpy's float32 cos differs by an ulp at times, which moves the IoU by up to 1e-5)"""
    c, s = F32(math.cos(float(b[4]))), F32(math.sin(float(b[4])))
    hx, hy = F32(b[2] * F32(0.5)), F32(b[3] * F32(0.5))
    xs, ys = (-hx, -hx, hx, hx), (-hy, hy, hy, -hy)
    out = []
    for i in range(4):
        out.append(F32(F32(c * xs[i]) + F32(s * ys[i])) + b[0])
        out.append(F32(F32(-s * xs[i]) + F32(c * ys[i])) + b[1])
    return out


def _in_quad(px, py, q):
    ab0, ab1 = q[2] - q[0], q[3] - q[1]
    ad0, ad1 = q[6] - q[0], q[7] - q[1]
    ap0, ap1 = px - q[0], py - q[1]
    abab, abap = ab0 * ab0 + ab1 * ab1, ab0 * ap0 + ab1 * ap1
    adad, adap = ad0 * ad0 + ad1 * ad1, ad0 * ap0 + ad1 * ap1
    return abab >= abap and abap >= 0 and adad >= adap and adap >= 0


def _seg(p1, p2, i, j):
    a0, a1 = p1[2 * i], p1[2 * i + 1]
    b0, b1 = p1[2 * ((i + 1) % 4)], p1[2 * ((i + 1) % 4) + 1]
    c0, c1 = p2[2 * j], p2[2 * j + 1]
    d0, d1 = p2[2 * ((j + 1) % 4)], p2[2 * ((j + 1) % 4) + 1]
    ba0, ba1, da0, ca0, da1, ca1 = b0 - a0, b1 - a1, d0 - a0, c0 - a0, d1 - a1, c1 - a1
    acd = da1 * ca0 > ca1 * da0
    bcd = (d1 - b1) * (c0 - b0) > (c1 - b1) * (d0 - b0)
    if acd != bcd:
        abc = ca1 * ba0 > ba1 * ca0
        abd = da1 * ba0 > ba1 * da0
        if abc != abd:
            dc0, dc1 = d0 - c0, d1 - c1
            abba = a0 * b1 - b0 * a1
            cddc = c0 * d1 - d0 * c1
            dh = ba1 * dc0 - ba0 * dc1
            return (abba * dc0 - ba0 * cddc) / dh, (abba * dc1 - ba1 * cddc) / dh
    return None


def _inter(b1, b2):
    """E2: the intersection area of two rotated boxes (b1 first, as the reference's kernel passes the query box first)"""
    with np.errstate(all='ignore'):
        p1, p2 = _corners(b1), _corners(b2)
        pts = []
        for i in range(4):
            if _in_quad(p1[2 * i], p1[2 * i + 1], p2):
                pts.append([p1[2 * i], p1[2 * i + 1]])
            if _in_quad(p2[2 * i], p2[2 * i + 1], p1):
                pts.append([p2[2 * i], p2[2 * i + 1]])
        for i in range(4):
            for j in range(4):
                r = _seg(p1, p2, i, j)
                if r is not None:
                    pts.append(list(r))
        n = len(pts)
        if n > 0:      # E3: sort by the pseudo-angle around the mean, insertion sort
            cx, cy = F32(0), F32(0)
            for p in pts:
                cx, cy = F32(cx + p[0]), F32(cy + p[1])
            cx, cy = F32(cx / F32(n)), F32(cy / F32(n))
            vs = []
            for p in pts:
                v0, v1 = F32(p[0] - cx), F32(p[1] - cy)
                d = F32(np.sqrt(F32(F32(v0 * v0) + F32(v1 * v1))))
                v0, v1 = F32(v0 / d), F32(v1 / d)
                if v1 < 0:
                    v0 = F32(F32(-2) - v0)
                vs.append(v0)
            for i in range(1, n):
                if vs[i - 1] > vs[i]:
                    t, tp = vs[i], pts[i]
                    j = i
                    while j > 0 and vs[j - 1] > t:
                        vs[j], pts[j] = vs[j - 1], pts[j - 1]
                        j -= 1
                    vs[j], pts[j] = t, tp
        area = 0.0     # E4: float64 sum of the float32 triangle areas
        for i in range(n - 2):
            a, b, c = pts[0], pts[i + 1], pts[i + 2]
            t = F32(F32((a[0] - c[0]) * (b[1] - c[1])) - F32((a[1] - c[1]) * (b[0] - c[0])))
            area += abs(float(t) / 2.0)
        return area


def rotate_iou(boxes, qboxes, criterion=-1):
    """rotate_iou_gpu_eval: [N, 5], [K, 5] -> float32 [N, K], entry (n, k) from the query box k and the box n"""
    b = np.asarray(boxes, np.float32).reshape(-1, 5)
    q = np.asarray(qboxes, np.float32).reshape(-1, 5)
    out = np.zeros((len(b), len(q)), np.float32)
    rb = np.hypot(b[:, 2], b[:, 3]).astype(np.float64) * 0.5
    rq = np.hypot(q[:, 2], q[:, 3]).astype(np.float64) * 0.5
    for n in range(len(b)):
        for k in range(len(q)):
            # boxes whose circumcircles are apart have no corner inside the other and no crossing edge: area 0
            if math.hypot(float(b[n, 0]) - float(q[k, 0]), float(b[n, 1]) - float(q[k, 1])) > rb[n] + rq[k] + 1e-3:
                continue
            inter = _inter(q[k], b[n])
            a1, a2 = F32(q[k, 2] * q[k, 3]), F32(b[n, 2] * b[n, 3])
            with np.errstate(all='ignore'):
                if criterion == -1:
                    out[n, k] = inter / (float(F32(a1 + a2)) - inter)
                elif criterion == 0:
                    out[n, k] = inter / float(a1)
                elif criterion == 1:
                    out[n, k] = inter / float(a2)
                else:
                    out[n, k] = inter
    return out


def image_iou(boxes, qboxes, criterion=-1):
    """image_box_overlap in float64: [N, 4], [K, 4] -> [N, K]"""
    b, q = np.asarray(boxes, np.float64), np.asarray(qboxes, np.float64)
    out = np.zeros((len(b), len(q)))
    for k in range(len(q)):
        qa = (q[k, 2] - q[k, 0]) * (q[k, 3] - q[k, 1])
        for n in range(len(b)):
            iw = min(b[n, 2], q[k, 2]) - max(b[n, 0], q[k, 0])
            if iw > 0:
                ih = min(b[n, 3], q[k, 3]) - max(b[n, 1], q[k, 1])
                if ih > 0:
                    ua = {-1: (b[n, 2] - b[n, 0]) * (b[n, 3] - b[n, 1]) + qa - iw * ih,
                          0: (b[n, 2] - b[n, 0]) * (b[n, 3] - b[n, 1]), 1: qa}.get(criterion, 1.0)
                    out[n, k] = iw * ih / ua
    return out


def _box7(a):
    return np.concatenate([a['location'], a['dimensions'], a['rotation_y'][:, None]], 1).astype(np.float64)


def frame_overlap(g, d, metric):
    """one frame's [n_dt, n_gt] float64 block of `metric` (0 image, 1 BEV, 2 3-D)"""
    if metric == 0:
        return image_iou(d['bbox'], g['bbox'])
    bd, bg = _box7(d), _box7(g)
    if metric == 1:
        return rotate_iou(bd[:, [0, 2, 3, 5, 6]], bg[:, [0, 2, 3, 5, 6]], -1).astype(np.float64)
    rinc = rotate_iou(bd[:, [0, 2, 3, 5, 6]], bg[:, [0, 2, 3, 5, 6]], 2)
    for i in range(len(bd)):
        for j in range(len(bg)):
            if rinc[i, j] > 0:
                iw = min(bd[i, 1], bg[j, 1]) - max(bd[i, 1] - bd[i, 4], bg[j, 1] - bg[j, 4])
                if iw > 0:
                    inc = iw * float(rinc[i, j])
                    rinc[i, j] = inc / (bd[i, 3] * bd[i, 4] * bd[i, 5] + bg[j, 3] * bg[j, 4] * bg[j, 5] - inc)
                else:
                    rinc[i, j] = 0.0
    return rinc.astype(np.float64)


def overlaps(gt_annos, dt_annos, metric):
    return [frame_overlap(g, d, metric) for g, d in zip(gt_annos, dt_annos)]


# ----------------------------------------------------------------------------------------------------------- ignore flags
def ignore_flags(g, d, cls, diff):
    """clean_data: (num_valid_gt, ignored_gt [n_gt], ignored_dt [n_dt], dontcare boxes [n_dc, 4])"""
    name = CLASS_NAMES[cls]
    ig = np.full(len(g['name']), -1, np.int64)
    for i, n in enumerate(g['name']):
        n = n.lower()
        valid = 1 if n == name else 0 if (name, n) in (('pedestrian', 'person_sitting'), ('car', 'van')) else -1
        h = g['bbox'][i, 3] - g['bbox'][i, 1]
        ignore = (g['occluded'][i] > MAX_OCCLUSION[diff] or g['truncated'][i] > MAX_TRUNCATION[diff]
                  or h <= MIN_HEIGHT[diff])
        ig[i] = 0 if (valid == 1 and not ignore) else 1 if (valid == 0 or (ignore and valid == 1)) else -1
    idt = np.empty(len(d['name']), np.int64)
    for j, n in enumerate(d['name']):
        h = abs(d['bbox'][j, 3] - d['bbox'][j, 1])
        idt[j] = 1 if h < MIN_HEIGHT[diff] else 0 if n.lower() == name else -1
    dc = np.array([g['bbox'][i] for i, n in enumerate(g['name']) if n == 'DontCare'], np.float64).reshape(-1, 4)
    return int((ig == 0).sum()), ig, idt, dc


# --------------------------------------------------------------------------------------------------------------- matching
NO_DET = -10000000


def match(ov, ig, idt, score, dt_alpha, gt_alpha, dc_ov, min_ov, thresh, compute_fp, metric, compute_aos):
    """compute_statistics_jit for one frame over L lanes: ov [L, n_dt, n_gt], ig [L, n_gt], idt [L, n_dt], dc_ov
    [n_dt, n_dc] (criterion-0 image overlap of the detections with the DontCare boxes), min_ov / thresh [L].
    -> tp, fp, fn [L] int, similarity [L] float64 (-1: none), matched [L, n_dt] bool (the detections counted as tp)"""
    L, nd, ng = ov.shape
    ar = np.arange(L)
    assigned = np.zeros((L, nd), bool)
    below = (score[None, :] < thresh[:, None]) if compute_fp else np.zeros((L, nd), bool)
    tp, fp, fn = np.zeros(L, np.int64), np.zeros(L, np.int64), np.zeros(L, np.int64)
    tp_det = np.zeros((L, nd), bool)
    sim = np.zeros(L)
    for i in range(ng):
        det = np.full(L, -1)
        valid = np.full(L, float(NO_DET))
        maxov = np.zeros(L)
        ass_ign = np.zeros(L, bool)
        for j in range(nd):
            live = (idt[:, j] != -1) & ~assigned[:, j] & ~below[:, j]
            o = ov[:, j, i]
            if not compute_fp:
                c = live & (o > min_ov) & (score[j] > valid)
                det = np.where(c, j, det)
                valid = np.where(c, score[j], valid)
            else:
                c1 = live & (o > min_ov) & ((o > maxov) | ass_ign) & (idt[:, j] == 0)
                c2 = live & ~c1 & (o > min_ov) & (valid == NO_DET) & (idt[:, j] == 1)
                maxov = np.where(c1, o, maxov)
                det = np.where(c1 | c2, j, det)
                valid = np.where(c1 | c2, 1.0, valid)
                ass_ign = np.where(c1, False, np.where(c2, True, ass_ign))
        act = ig[:, i] != -1
        none = valid == NO_DET
        dsafe = np.maximum(det, 0)
        fn += act & none & (ig[:, i] == 0)
        idt_det = idt[ar, dsafe] if nd else np.zeros(L, np.int64)
        ign_match = act & ~none & ((ig[:, i] == 1) | (idt_det == 1))
        is_tp = act & ~none & ~ign_match
        tp += is_tp
        assigned[ar[ign_match | is_tp], dsafe[ign_match | is_tp]] = True
        tp_det[ar[is_tp], dsafe[is_tp]] = True
        if compute_aos:
            if nd:
                sim = np.where(is_tp, sim + (1.0 + np.cos(gt_alpha[i] - dt_alpha[dsafe])) / 2.0, sim)
    if compute_fp:
        fp = (~(assigned | (idt == -1) | (idt == 1) | below)).sum(1)
        if metric == 0:
            nstuff = np.zeros(L, np.int64)
            for k in range(dc_ov.shape[1]):
                for j in range(nd):
                    c = ~assigned[:, j] & (idt[:, j] == 0) & ~below[:, j] & (dc_ov[j, k] > min_ov)
                    assigned[:, j] |= c
                    nstuff += c
            fp = fp - nstuff
        if compute_aos:
            sim = np.where((tp > 0) | (fp > 0), sim, -1.0)
    return tp, fp, fn, sim, tp_det


def thresholds(scores, num_gt):
    """get_thresholds: the 41-point selection over the scores sorted high to low"""
    s = np.sort(np.asarray(scores, np.float64))[::-1]
    cur, out = 0.0, []
    for i, v in enumerate(s):
        lr = (i + 1) / num_gt
        rr = (i + 2) / num_gt if i < len(s) - 1 else lr
        if (rr - cur) < (cur - lr) and i < len(s) - 1:
            continue
        out.append(v)
        cur += 1 / (N_SAMPLE_PTS - 1.0)
    return np.array(out, np.float64)


def evaluate(gt_annos, dt_annos, classes, min_overlaps, compute_aos, metrics=(0, 1, 2)):
    """eval_class for each metric.  min_overlaps [K, 3, C] (already indexed by `classes`).  Returns per metric m:
    overlaps[m] (list of per-frame blocks), thresholds[m][c][d][k], pr[m][c][d][k] ([T, 4]: tp, fp, fn, similarity),
    precision / recall / orientation [m] ([C, 3, K, 41])."""
    F = len(gt_annos)
    C, K = len(classes), min_overlaps.shape[0]
    lanes = [(c, d, k) for c in range(C) for d in range(3) for k in range(K)]
    flags = [[[ignore_flags(gt_annos[f], dt_annos[f], classes[c], d) for f in range(F)] for d in range(3)]
             for c in range(C)]
    dc_ov = [image_iou(dt_annos[f]['bbox'], flags[0][0][f][3], 0) for f in range(F)]
    res = {'overlaps': {}, 'thresholds': {}, 'pr': {}, 'precision': {}, 'recall': {}, 'orientation': {}}
    for m in metrics:
        ovs = overlaps(gt_annos, dt_annos, m)
        res['overlaps'][m] = ovs
        aos_m = compute_aos and m == 0
        mo = np.array([min_overlaps[k, m, c] for c, d, k in lanes])
        # pass 1: thresh 0, no false positives; the scores of the true positives
        tps = [[] for _ in lanes]
        for f in range(F):
            g, dd = gt_annos[f], dt_annos[f]
            ig = np.stack([flags[c][d][f][1] for c, d, k in lanes])
            idt = np.stack([flags[c][d][f][2] for c, d, k in lanes])
            ov = np.broadcast_to(ovs[f], (len(lanes),) + ovs[f].shape)
            _, _, _, _, hit = match(ov, ig, idt, dd['score'].astype(np.float64), None, None, dc_ov[f], mo,
                                    np.zeros(len(lanes)), False, m, False)
            for li in range(len(lanes)):
                tps[li].extend(dd['score'].astype(np.float64)[hit[li]].tolist())
        ths = [thresholds(tps[li], sum(flags[c][d][f][0] for f in range(F))) for li, (c, d, k) in enumerate(lanes)]
        # pass 2: every threshold of every lane
        sub = [(li, t) for li in range(len(lanes)) for t in range(len(ths[li]))]
        pr = [np.zeros((len(ths[li]), 4)) for li in range(len(lanes))]
        if sub:
            li_of = np.array([s[0] for s in sub])
            th = np.array([ths[li][t] for li, t in sub])
            for f in range(F):
                g, dd = gt_annos[f], dt_annos[f]
                ig = np.stack([flags[lanes[li][0]][lanes[li][1]][f][1] for li in li_of])
                idt = np.stack([flags[lanes[li][0]][lanes[li][1]][f][2] for li in li_of])
                ov = np.broadcast_to(ovs[f], (len(sub),) + ovs[f].shape)
                tp, fp, fn, sim, _ = match(ov, ig, idt, dd['score'].astype(np.float64), dd['alpha'].astype(np.float64),
                                           g['alpha'].astype(np.float64), dc_ov[f], mo[li_of], th, True, m, aos_m)
                for s, (li, t) in enumerate(sub):
                    pr[li][t, 0] += tp[s]
                    pr[li][t, 1] += fp[s]
                    pr[li][t, 2] += fn[s]
                    if aos_m and sim[s] != -1:
                        pr[li][t, 3] += sim[s]
        prec, rec, aos = np.zeros((3, C, 3, K, N_SAMPLE_PTS))
        with np.errstate(all='ignore'):
            for li, (c, d, k) in enumerate(lanes):
                p = pr[li]
                for i in range(len(p)):
                    rec[c, d, k, i] = p[i, 0] / (p[i, 0] + p[i, 2])
                    prec[c, d, k, i] = p[i, 0] / (p[i, 0] + p[i, 1])
                    if aos_m:
                        aos[c, d, k, i] = p[i, 3] / (p[i, 0] + p[i, 1])
                for i in range(len(p)):
                    prec[c, d, k, i] = np.max(prec[c, d, k, i:])
                    if aos_m:
                        aos[c, d, k, i] = np.max(aos[c, d, k, i:])
        res['thresholds'][m] = {lanes[li]: ths[li] for li in range(len(lanes))}
        res['pr'][m] = {lanes[li]: pr[li] for li in range(len(lanes))}
        res['precision'][m], res['recall'][m], res['orientation'][m] = prec, rec, aos
    return res


# ------------------------------------------------------------------------------------------------ synthetic annotations
_SIZES = {'Car': (3.9, 1.56, 1.6), 'Van': (5.0, 2.1, 1.9), 'Truck': (10.0, 3.2, 2.6), 'Pedestrian': (0.8, 1.75, 0.6),
          'Person_sitting': (0.8, 1.25, 0.6), 'Cyclist': (1.76, 1.73, 0.6)}
_DET_NAME = {'Car': 'Car', 'Van': 'Car', 'Truck': 'Car', 'Pedestrian': 'Pedestrian', 'Person_sitting': 'Pedestrian',
             'Cyclist': 'Cyclist'}
_FOCAL, _CU, _CV = 721.5377, 609.5593, 172.854      # KITTI P2


def _anno(names, trunc, occ, alpha, bbox, dims, loc, rot, score=None):
    n = len(names)
    a = {'name': np.array(names, dtype='<U14'), 'truncated': np.array(trunc, np.float64).reshape(n),
         'occluded': np.array(occ, np.int64).reshape(n), 'alpha': np.array(alpha, np.float64).reshape(n),
         'bbox': np.array(bbox, np.float64).reshape(n, 4), 'dimensions': np.array(dims, np.float64).reshape(n, 3),
         'location': np.array(loc, np.float64).reshape(n, 3), 'rotation_y': np.array(rot, np.float64).reshape(n)}
    a['score'] = np.zeros(n, np.float64) if score is None else np.array(score, np.float32).reshape(n)
    return a


def _project(x, y, z, l, h, w):
    """a 2-D box around the object's image footprint (bottom centre at (x, y, z), camera frame)"""
    r = 0.5 * max(l, w)
    u0, u1 = _FOCAL * (x - r) / z + _CU, _FOCAL * (x + r) / z + _CU
    v0, v1 = _FOCAL * (y - h) / z + _CV, _FOCAL * y / z + _CV
    return [max(0.0, u0), max(0.0, v0), min(1241.0, u1), min(374.0, v1)]


def _obj(rng, name):
    l, h, w = (s * rng.uniform(0.9, 1.1) for s in _SIZES[name])
    z = rng.uniform(4.0, 55.0)
    x = rng.uniform(-0.6, 0.6) * z
    y = rng.uniform(1.4, 1.9)
    ry = rng.uniform(-np.pi, np.pi)
    return [x, y, z], [l, h, w], ry


def _frame(rng, n_gt, p_dc, with_alpha):
    kinds = ['Car', 'Car', 'Car', 'Car', 'Pedestrian', 'Pedestrian', 'Cyclist', 'Van', 'Person_sitting', 'Truck']
    g = {k: [] for k in ('names', 'trunc', 'occ', 'alpha', 'bbox', 'dims', 'loc', 'rot')}
    d = {k: [] for k in ('names', 'alpha', 'bbox', 'dims', 'loc', 'rot', 'score')}

    def add_det(name, loc, dims, ry, bbox):
        d['names'].append(name)
        d['loc'].append(loc)
        d['dims'].append(dims)
        d['rot'].append(ry)
        d['bbox'].append(bbox)
        d['alpha'].append(ry - math.atan2(loc[0], loc[2]) + rng.normal(0, 0.2) if with_alpha else -10.0)
        d['score'].append(rng.uniform(0.02, 1.0))

    for _ in range(n_gt):
        if rng.uniform() < p_dc:
            u, v = rng.uniform(0, 1100), rng.uniform(120, 220)
            for k, val in (('names', 'DontCare'), ('trunc', -1.0), ('occ', -1), ('alpha', -10.0),
                           ('bbox', [u, v, u + rng.uniform(10, 140), v + rng.uniform(10, 60)]),
                           ('dims', [-1.0, -1.0, -1.0]), ('loc', [-1000.0, -1000.0, -1000.0]), ('rot', -10.0)):
                g[k].append(val)
            continue
        name = kinds[rng.integers(len(kinds))]
        loc, dims, ry = _obj(rng, name)
        bbox = _project(*loc, *dims)
        g['names'].append(name)
        g['trunc'].append(float(rng.choice([0.0, 0.0, 0.1, 0.2, 0.4, 0.7])))
        g['occ'].append(int(rng.integers(0, 4)))
        g['alpha'].append(ry - math.atan2(loc[0], loc[2]))
        g['bbox'].append(bbox)
        g['dims'].append(dims)
        g['loc'].append(loc)
        g['rot'].append(ry)
        if rng.uniform() < 0.85:        # detected: jittered box, score
            dl = [loc[0] + rng.normal(0, 0.25), loc[1] + rng.normal(0, 0.08), loc[2] + rng.normal(0, 0.35)]
            dd = [s * rng.uniform(0.92, 1.08) for s in dims]
            dr = ry + rng.normal(0, 0.12)
            add_det(_DET_NAME[name], dl, dd, dr, [c + rng.normal(0, 4.0) for c in bbox])
            if rng.uniform() < 0.1:     # a duplicate
                add_det(_DET_NAME[name], [c + rng.normal(0, 0.4) for c in dl], dd, dr, [c + rng.normal(0, 8.0) for c in bbox])
    for _ in range(int(rng.integers(0, 3))):      # false positives
        name = ['Car', 'Pedestrian', 'Cyclist'][rng.integers(3)]
        loc, dims, ry = _obj(rng, name)
        add_det(name, loc, dims, ry, _project(*loc, *dims))
    gt = _anno(g['names'], g['trunc'], g['occ'], g['alpha'], g['bbox'], g['dims'], g['loc'], g['rot'])
    dt = _anno(d['names'], [0.0] * len(d['names']), [0] * len(d['names']), d['alpha'], d['bbox'], d['dims'], d['loc'],
               d['rot'], d['score'])
    return gt, dt


# min-overlap values of the official and the COCO-style evaluation
MIN_OVERLAP_VALUES = sorted({0.25, 0.5, 0.7} | {round(v, 10) for v in np.linspace(0.5, 0.95, 10)}
                            | {round(v, 10) for v in np.linspace(0.25, 0.7, 10)})
NEAR = 1e-5


def near_threshold(g, d):
    """True where an overlap of the frame (any metric, or a detection's overlap with a DontCare box) lies within NEAR
    of a min-overlap value: float32 rounding differences could flip such a match"""
    blocks = [frame_overlap(g, d, m) for m in range(3)]
    dc = np.array([g['bbox'][i] for i, n in enumerate(g['name']) if n == 'DontCare'], np.float64).reshape(-1, 4)
    blocks.append(image_iou(d['bbox'], dc, 0))
    vals = np.concatenate([b.ravel() for b in blocks])
    return bool(np.any(np.abs(vals[:, None] - np.array(MIN_OVERLAP_VALUES)[None, :]) < NEAR))


def synthetic_annos(seed, n_frames, max_gt=12, p_dc=0.1, with_alpha=True, check_near=True, empty=()):
    """seeded KITTI-style (gt_annos, dt_annos): cars, vans, trucks, pedestrians, sitting persons, cyclists and DontCare
    boxes with truncation and occlusion; detections jittered, dropped, duplicated and added, float32 scores.  A frame
    with an overlap near a min-overlap value is drawn again (check_near).  `empty`: frame indices with neither GT nor
    detections."""
    rng = np.random.default_rng(seed)
    gts, dts = [], []
    for f in range(n_frames):
        while True:
            gt, dt = _frame(rng, 0 if f in empty else int(rng.integers(0, max_gt + 1)), p_dc, with_alpha)
            if f in empty:
                dt = _anno([], [], [], [], [], [], [], [], [])
            if not check_near or not near_threshold(gt, dt):
                break
        gts.append(gt)
        dts.append(dt)
    return gts, dts
