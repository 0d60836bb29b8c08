"""KITTI evaluation on the sm_90a kernels of csrc/kitti_eval.cu (geometry rules in csrc/kitti_eval_geom.cuh): the AP
tables of kitti_object_eval_python/eval.py for a whole evaluation set from one upload, nine launches and one read-back.

  * `get_official_eval_result(gt_annos, dt_annos, current_classes, PR_detail_dict=None)` -> (result_str, ret_dict),
    drop-in for eval.py's function of the same name (the string and the `Car_3d/moderate_R40`-style keys as it forms them);
  * `get_coco_eval_result(gt_annos, dt_annos, current_classes)` -> result_str, the COCO-style mean over 10 min-overlap
    values per class;
  * `eval_overlaps(gt_annos, dt_annos, metric)` -> the per-frame [n_dt, n_gt] overlap blocks of one metric (0 image,
    1 BEV, 2 3-D), as calculate_iou_partly(dt_annos, gt_annos, metric)[0] lists them;
  * `rotate_iou_eval(boxes, qboxes, criterion=-1, device_id=0)` -> float32 [N, K], drop-in for rotate_iou_gpu_eval.

Annotations are packed on the host into float64 rows (include/virconv_b200.h, VC_KE_ROW) and uploaded in one copy; the
tables come back in one copy, and the R11 / R40 means and the string are formed on the host.  There is no CPU path: the
kernels are the implementation."""
from __future__ import annotations

import io

import numpy as np
import torch

from . import _lib, ops
from ._lib import check

ROW = 16
SAMPLES = 41
LANE_W = 329
CLASS_TO_NAME = {0: 'Car', 1: 'Pedestrian', 2: 'Cyclist', 3: 'Van', 4: 'Person_sitting', 5: 'Truck'}
_CLASS_ID = {'car': 0, 'pedestrian': 1, 'cyclist': 2, 'van': 3, 'person_sitting': 4, 'truck': 5}
# [overlap setting, metric (bbox, bev, 3d), class 0..5]: eval.py's overlap_0_7 and overlap_0_5
_OFFICIAL_MIN_OVERLAPS = np.array([[[0.7, 0.5, 0.5, 0.7, 0.5, 0.7]] * 3,
                                   [[0.7, 0.5, 0.5, 0.7, 0.5, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5],
                                    [0.5, 0.25, 0.25, 0.5, 0.25, 0.5]]])
_COCO_RANGE = {0: (0.5, 0.95, 10), 1: (0.25, 0.7, 10), 2: (0.25, 0.7, 10), 3: (0.5, 0.95, 10), 4: (0.25, 0.7, 10)}


def _class_ids(current_classes, names):
    if not isinstance(current_classes, (list, tuple)):
        current_classes = [current_classes]
    rev = {v: k for k, v in names.items()}
    out = [rev[c] if isinstance(c, str) else int(c) for c in current_classes]
    for c in out:
        if c not in names:
            raise KeyError(c)
    return out


def _compute_aos(dt_annos):
    """eval.py's test: the first detection of the first frame with any detection has an alpha other than -10"""
    for a in dt_annos:
        if a['alpha'].shape[0] != 0:
            return bool(a['alpha'][0] != -10)
    return False


def pack(gt_annos, dt_annos):
    """annotation dicts -> (gt rows [NG, 16], dt rows [ND, 16], offs int64 [3, F + 1], n_pair)"""
    if len(gt_annos) != len(dt_annos):
        raise ValueError(f'{len(gt_annos)} GT frames and {len(dt_annos)} detection frames')
    ng = np.array([len(a['name']) for a in gt_annos], np.int64)
    nd = np.array([len(a['name']) for a in dt_annos], np.int64)
    for what, annos, n in (('gt', gt_annos, ng), ('dt', dt_annos, nd)):
        for f, a in enumerate(annos):
            for k, w in (('bbox', 4), ('location', 3), ('dimensions', 3)):
                if np.shape(a[k]) != (n[f], w):
                    raise ValueError(f'{what}_annos[{f}][{k!r}] has shape {np.shape(a[k])}, expected ({n[f]}, {w})')
            for k in ('alpha', 'rotation_y') + (('truncated', 'occluded') if what == 'gt' else ('score',)):
                if np.shape(a[k]) != (n[f],):
                    raise ValueError(f'{what}_annos[{f}][{k!r}] has shape {np.shape(a[k])}, expected ({n[f]},)')

    def rows(annos, n, extra):
        out = np.zeros((int(n.sum()), ROW), np.float64)
        if len(out) == 0:
            return out
        cat = lambda k, w=1: np.concatenate([np.asarray(a[k], np.float64).reshape(len(a['name']), w) for a in annos], 0)
        out[:, 0:4] = cat('bbox', 4)
        out[:, 4] = cat('alpha')[:, 0]
        out[:, 5:8] = cat('location', 3)
        out[:, 8:11] = cat('dimensions', 3)
        out[:, 11] = cat('rotation_y')[:, 0]
        names = [str(s) for a in annos for s in a['name']]
        cls = np.array([_CLASS_ID.get(s.lower(), -1) for s in names], np.float64)
        if extra == 'gt':
            out[:, 12] = cat('truncated')[:, 0]
            out[:, 13] = cat('occluded')[:, 0]
            out[:, 14] = cls
            out[:, 15] = np.array([s == 'DontCare' for s in names], np.float64)
        else:
            out[:, 12] = cat('score')[:, 0]
            out[:, 13] = cls
        return out

    offs = np.zeros((3, len(ng) + 1), np.int64)
    offs[0, 1:] = np.cumsum(ng)
    offs[1, 1:] = np.cumsum(nd)
    offs[2, 1:] = np.cumsum(ng * nd)
    return rows(gt_annos, ng, 'gt'), rows(dt_annos, nd, 'dt'), offs, int(offs[2, -1])


def _upload(arrays, device):
    """one host-to-device copy of the arrays (8-byte aligned), returns the buffer and each array's device address"""
    blob = np.concatenate([np.ascontiguousarray(a).view(np.uint8).ravel() for a in arrays])
    buf = torch.from_numpy(blob).to(device)
    ptrs, off = [], 0
    for a in arrays:
        ptrs.append(buf.data_ptr() + off)
        off += a.nbytes
    return buf, ptrs


def _device(device):
    if device is None:
        if not torch.cuda.is_available():
            raise RuntimeError('virconv_b200.kitti_eval needs a CUDA device')
        return torch.device('cuda', torch.cuda.current_device())
    return torch.device(device)


def eval_tables(gt_annos, dt_annos, classes, min_overlaps, compute_aos, device=None, return_overlaps=False):
    """eval_class for metrics 0, 1, 2.  classes: class ids; min_overlaps [K, 3, len(classes)].  Returns a dict of numpy
    arrays indexed [metric, class, difficulty, overlap setting, ...]: 'n_thresholds', 'thresholds' [.., 41], 'pr'
    [.., 41, 4] (tp, fp, fn, similarity), 'precision', 'recall', 'orientation' [.., 41]; with return_overlaps also
    'overlaps' [3, n_pair] and 'offs'."""
    classes = [int(c) for c in classes]
    mo = np.asarray(min_overlaps, np.float64)
    C, K = len(classes), mo.shape[0]
    if not 1 <= C <= 6 or any(not 0 <= c <= 5 for c in classes):
        raise ValueError(f'classes {classes}: 1 to 6 class ids in 0..5')
    if mo.shape != (K, 3, C) or not 1 <= K <= 10:
        raise ValueError(f'min_overlaps of shape {mo.shape}, expected (K, 3, {C}) with 1 <= K <= 10')
    gt, dt, offs, P = pack(gt_annos, dt_annos)
    F, NG, ND = offs.shape[1] - 1, len(gt), len(dt)
    L = 3 * C * 3 * K
    lane_mo = np.array([mo[k, m, c] for m in range(3) for c in range(C) for d in range(3) for k in range(K)], np.float64)
    dev = _device(device)
    lib = _lib.load()
    with torch.cuda.device(dev):
        buf, (p_gt, p_dt, p_offs, p_mo) = _upload([gt, dt, offs, lane_mo], dev)
        ov = torch.empty(max(3 * P, 1), dtype=torch.float64, device=dev)
        out = torch.empty(L * LANE_W, dtype=torch.float64, device=dev)
        wsb = lib.vc_kitti_eval_ws_bytes(F, NG, ND, C, K)
        ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=dev)
        check(lib.vc_kitti_eval(p_gt, p_dt, p_offs, p_mo, F, NG, ND, P, C, _lib.host_i32(classes), K, int(compute_aos),
                                ov.data_ptr(), out.data_ptr(), ws.data_ptr(), wsb, ops._stream()), 'vc_kitti_eval')
        o = out.cpu().numpy().reshape(3, C, 3, K, LANE_W)
        res = {'n_thresholds': o[..., 0].astype(np.int64), 'thresholds': o[..., 1:1 + SAMPLES],
               'pr': o[..., 1 + SAMPLES:1 + 5 * SAMPLES].reshape(3, C, 3, K, SAMPLES, 4),
               'precision': o[..., 1 + 5 * SAMPLES:1 + 6 * SAMPLES], 'recall': o[..., 1 + 6 * SAMPLES:1 + 7 * SAMPLES],
               'orientation': o[..., 1 + 7 * SAMPLES:1 + 8 * SAMPLES]}
        if return_overlaps:
            res['overlaps'] = ov[:3 * P].cpu().numpy().reshape(3, P)
            res['offs'] = offs
        del buf
    return res


def eval_overlaps(gt_annos, dt_annos, metric, device=None):
    """the per-frame [n_dt, n_gt] float64 overlap blocks of `metric` (0 image, 1 BEV, 2 3-D)"""
    if metric not in (0, 1, 2):
        raise ValueError(f'metric {metric}: 0 (image), 1 (BEV) or 2 (3-D)')
    gt, dt, offs, P = pack(gt_annos, dt_annos)
    F = offs.shape[1] - 1
    dev = _device(device)
    with torch.cuda.device(dev):
        buf, (p_gt, p_dt, p_offs) = _upload([gt, dt, offs], dev)
        ov = torch.empty(max(P, 1), dtype=torch.float64, device=dev)
        check(_lib.load().vc_kitti_overlaps(p_gt, p_dt, p_offs, F, P, metric, ov.data_ptr(), ops._stream()),
              'vc_kitti_overlaps')
        flat = ov[:P].cpu().numpy()
    ng, nd = np.diff(offs[0]), np.diff(offs[1])
    return [flat[offs[2, f]:offs[2, f + 1]].reshape(nd[f], ng[f]) for f in range(F)]


def rotate_iou_eval(boxes, query_boxes, criterion=-1, device_id=0):
    """rotate_iou_gpu_eval: boxes [N, 5], query_boxes [K, 5] (x, y, dx, dy, angle) -> float32 numpy [N, K]; entry
    (n, k) is the overlap of query box k with box n under `criterion` (-1 IoU, 0 / 1 over the query / box area, 2 the
    intersection)"""
    b = np.ascontiguousarray(np.asarray(boxes, np.float32).reshape(-1, 5))
    q = np.ascontiguousarray(np.asarray(query_boxes, np.float32).reshape(-1, 5))
    N, K = len(b), len(q)
    if N == 0 or K == 0:
        return np.zeros((N, K), np.float32)
    dev = torch.device('cuda', device_id)
    with torch.cuda.device(dev):
        buf, (pb, pq) = _upload([b, q], dev)
        out = torch.empty(N * K, dtype=torch.float32, device=dev)
        check(_lib.load().vc_kitti_rotate_iou(pb, pq, N, K, int(criterion), out.data_ptr(), ops._stream()),
              'vc_kitti_rotate_iou')
        return out.cpu().numpy().reshape(N, K)


def get_mAP(prec):
    s = 0
    for i in range(0, prec.shape[-1], 4):
        s = s + prec[..., i]
    return s / 11 * 100


def get_mAP_R40(prec):
    s = 0
    for i in range(1, prec.shape[-1]):
        s = s + prec[..., i]
    return s / 40 * 100


def _line(text):
    buf = io.StringIO()
    print(text, file=buf)
    return buf.getvalue()


def _aps(gt_annos, dt_annos, classes, min_overlaps, compute_aos, PR_detail_dict=None):
    """(11-point, R40) mAP per metric name, each [C, 3, K]; aos entries None without AOS"""
    t = eval_tables(gt_annos, dt_annos, classes, min_overlaps, compute_aos)
    prec = t['precision']
    ap11 = {n: get_mAP(prec[m]) for m, n in enumerate(('bbox', 'bev', '3d'))}
    ap40 = {n: get_mAP_R40(prec[m]) for m, n in enumerate(('bbox', 'bev', '3d'))}
    ap11['aos'] = ap40['aos'] = None
    if compute_aos:
        ap11['aos'], ap40['aos'] = get_mAP(t['orientation'][0]), get_mAP_R40(t['orientation'][0])
    if PR_detail_dict is not None:
        PR_detail_dict['bbox'] = prec[0]
        if compute_aos:
            PR_detail_dict['aos'] = t['orientation'][0]
        PR_detail_dict['bev'] = prec[1]
        PR_detail_dict['3d'] = prec[2]
    return ap11, ap40


def get_official_eval_result(gt_annos, dt_annos, current_classes, PR_detail_dict=None):
    """KITTI AP at the official min overlaps: (result_str, ret_dict) as eval.py's get_official_eval_result forms them"""
    classes = _class_ids(current_classes, CLASS_TO_NAME)
    mo = _OFFICIAL_MIN_OVERLAPS[:, :, classes]
    compute_aos = _compute_aos(dt_annos)
    ap11, ap40 = _aps(gt_annos, dt_annos, classes, mo, compute_aos, PR_detail_dict)
    result, ret = '', {}
    rows = (('bbox AP', 'bbox'), ('bev  AP', 'bev'), ('3d   AP', '3d'))
    for j, c in enumerate(classes):
        name = CLASS_TO_NAME[c]
        for i in range(mo.shape[0]):
            for tag, ap in (('AP', ap11), ('AP_R40', ap40)):
                result += _line(f'{name} {tag}@' + '{:.2f}, {:.2f}, {:.2f}:'.format(*mo[i, :, j]))
                for label, key in rows:
                    result += _line(f'{label}:{ap[key][j, 0, i]:.4f}, {ap[key][j, 1, i]:.4f}, {ap[key][j, 2, i]:.4f}')
                if compute_aos:
                    a = ap['aos']
                    result += _line(f'aos  AP:{a[j, 0, i]:.2f}, {a[j, 1, i]:.2f}, {a[j, 2, i]:.2f}')
            if compute_aos and i == 0:
                for d, dn in enumerate(('easy', 'moderate', 'hard')):
                    ret[f'{name}_aos/{dn}_R40'] = ap40['aos'][j, d, 0]
            if i == 0:
                for key, kn in (('3d', '3d'), ('bev', 'bev'), ('bbox', 'image')):
                    for d, dn in enumerate(('easy', 'moderate', 'hard')):
                        ret[f'{name}_{kn}/{dn}_R40'] = ap40[key][j, d, 0]
    return result, ret


def get_coco_eval_result(gt_annos, dt_annos, current_classes):
    """COCO-style KITTI AP: the 11-point AP averaged over 10 min overlaps per class (0.5:0.05:0.95 for cars and vans,
    0.25:0.05:0.7 otherwise) -> result_str.  (eval.py's own get_coco_eval_result stops at unpacking do_eval's eight
    results into four; this is what its do_coco_style_eval computes with the first four.)"""
    names = {k: v for k, v in CLASS_TO_NAME.items() if k in _COCO_RANGE}
    classes = _class_ids(current_classes, names)
    mo = np.zeros((10, 3, len(classes)))
    for j, c in enumerate(classes):
        mo[:, :, j] = np.linspace(*_COCO_RANGE[c])[:, None]
    compute_aos = _compute_aos(dt_annos)
    ap11, _ = _aps(gt_annos, dt_annos, classes, mo, compute_aos)
    mean = {k: (None if v is None else v.mean(-1)) for k, v in ap11.items()}
    result = ''
    for j, c in enumerate(classes):
        r = np.array(_COCO_RANGE[c])[[0, 2, 1]]
        r[1] = (r[2] - r[0]) / (r[1] - 1)
        result += _line(f'{CLASS_TO_NAME[c]} coco AP@' + '{:.2f}:{:.2f}:{:.2f}:'.format(*r))
        for label, key in (('bbox AP', 'bbox'), ('bev  AP', 'bev'), ('3d   AP', '3d')) + (
                (('aos  AP', 'aos'),) if compute_aos else ()):
            result += _line(f'{label}:{mean[key][j, 0]:.2f}, {mean[key][j, 1]:.2f}, {mean[key][j, 2]:.2f}')
    return result
