"""Record what the reference's OWN KITTI evaluation (kitti_object_eval_python/eval.py: get_official_eval_result) returns
on seeded synthetic annotations, as tests/golden/kitti_eval_ref.npz.  Needs the reference's sources (imported through
virconv_b200.reference_env) and numba; the rotated-box kernel (rotate_iou.py, a numba CUDA kernel) runs under numba's
CUDA simulator on the CPU (NUMBA_ENABLE_CUDASIM=1, set here before numba is imported).  The fixture is committed, so
the tests need neither.

Besides `result_str` and `ret_dict`, the reference's intermediate results are recorded by wrapping three of the eval
module's functions: calculate_iou_partly (the per-frame [n_dt, n_gt] overlap blocks), get_thresholds (the 41-point
thresholds) and fused_compute_statistics (the tp / fp / fn / similarity table it fills per threshold).

Cases (oracle.kitti_eval.synthetic_annos; no overlap within 1e-5 of a min-overlap value):
  main  — 60 frames, up to 12 objects, 10 % DontCare, alphas valid (AOS computed), classes Car, Pedestrian, Cyclist;
  noaos — 16 frames, detection alphas -10 (no AOS), classes 'Car' given by name;
  edge  — 14 frames: frames 0, 5 and 9 empty, frames 2 and 7 DontCare only, no Cyclist GT anywhere, classes 0, 1, 2;
  nodet — 8 frames with GT and no detection at all.

    python -m oracle.kitti_eval_golden REFERENCE_ROOT [OUT_DIR]
"""
from __future__ import annotations

import os
import sys

os.environ['NUMBA_ENABLE_CUDASIM'] = '1'

import numpy as np   # noqa: E402

from oracle import kitti_eval as K   # noqa: E402

CASES = ('main', 'noaos', 'edge', 'nodet')


def case_annos(name):
    if name == 'main':
        return K.synthetic_annos(11, 60), [0, 1, 2]
    if name == 'noaos':
        return K.synthetic_annos(12, 16, with_alpha=False), 'Car'
    if name == 'edge':
        g, d = K.synthetic_annos(13, 14, empty=(0, 5, 9))
        for f in range(len(g)):
            keep = np.array([n not in ('Cyclist',) for n in g[f]['name']], bool)
            if f in (2, 7):
                keep &= g[f]['name'] == 'DontCare'
            g[f] = {k: v[keep] for k, v in g[f].items()}
        return (g, d), [0, 1, 2]
    if name == 'nodet':
        g, d = K.synthetic_annos(14, 8)
        d = [{k: v[:0] for k, v in a.items()} for a in d]
        return (g, d), [0, 1, 2]
    raise KeyError(name)


def pack_annos(prefix, annos, out):
    """annotation dicts -> flat arrays (names as one '|'-joined string per frame list)"""
    out[prefix + '.n'] = np.array([len(a['name']) for a in annos], np.int64)
    out[prefix + '.name'] = np.array('|'.join(n for a in annos for n in a['name']))
    for k in ('truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location', 'rotation_y', 'score'):
        out[prefix + '.' + k] = np.concatenate([a[k] for a in annos], 0)


def unpack_annos(prefix, z):
    n = z[prefix + '.n']
    names = str(z[prefix + '.name']).split('|') if int(n.sum()) else []
    off = np.concatenate([[0], np.cumsum(n)])
    return [{'name': np.array(names[off[f]:off[f + 1]], dtype='<U14'),
             **{k: z[prefix + '.' + k][off[f]:off[f + 1]] for k in
                ('truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location', 'rotation_y', 'score')}}
            for f in range(len(n))]


def make(reference_root, out_dir):
    from virconv_b200 import reference_env
    reference_env.install(reference_root=reference_root)
    import importlib
    ev = importlib.import_module('pcdet.datasets.kitti.kitti_object_eval_python.eval')
    rec = {}
    orig = {k: getattr(ev, k) for k in ('calculate_iou_partly', 'get_thresholds', 'fused_compute_statistics')}

    def calculate_iou_partly(gt_annos, dt_annos, metric, num_parts=50):
        r = orig['calculate_iou_partly'](gt_annos, dt_annos, metric, num_parts)
        rec['ov'].append(np.concatenate([o.ravel() for o in r[0]]) if r[0] else np.zeros(0))
        return r

    def get_thresholds(scores, num_gt, num_sample_pts=41):
        t = orig['get_thresholds'](scores, num_gt, num_sample_pts)
        rec['th'].append(np.array(t, np.float64))
        return t

    def fused_compute_statistics(overlaps, pr, *a, **kw):
        if not rec['pr'] or rec['pr'][-1] is not pr:
            rec['pr'].append(pr)
        return orig['fused_compute_statistics'](overlaps, pr, *a, **kw)

    ev.calculate_iou_partly, ev.get_thresholds = calculate_iou_partly, get_thresholds
    ev.fused_compute_statistics = fused_compute_statistics
    out = {}
    for case in CASES:
        (g, d), classes = case_annos(case)
        rec.update(ov=[], th=[], pr=[])
        pr_detail = {}
        s, rd = ev.get_official_eval_result(g, d, classes, PR_detail_dict=pr_detail)
        assert len(rec['ov']) == 3 and len(rec['th']) == len(rec['pr']), (len(rec['ov']), len(rec['th']), len(rec['pr']))
        pack_annos(case + '.gt', g, out)
        pack_annos(case + '.dt', d, out)
        out[case + '.classes'] = np.array(classes if isinstance(classes, list) else [classes], dtype='<U10')
        for m in range(3):
            out[f'{case}.ov{m}'] = rec['ov'][m]
        # thresholds and pr tables in the reference's loop order: metric, class, difficulty, overlap setting
        out[case + '.th_n'] = np.array([len(t) for t in rec['th']], np.int64)
        out[case + '.th'] = np.concatenate(rec['th']) if rec['th'] else np.zeros(0)
        out[case + '.pr'] = np.concatenate(rec['pr'], 0) if rec['pr'] else np.zeros((0, 4))
        out[case + '.result_str'] = np.array(s)
        out[case + '.ret_keys'] = np.array(list(rd.keys()))
        out[case + '.ret_vals'] = np.array([float(v) for v in rd.values()], np.float64)
        for k, v in pr_detail.items():
            out[f'{case}.prec_{k}'] = v
        print(case, sum(len(a['name']) for a in g), 'GT', sum(len(a['name']) for a in d), 'DT', flush=True)
        print(s)
    for k, v in orig.items():
        setattr(ev, k, v)
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'kitti_eval_ref.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    root = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    make(root, sys.argv[2] if len(sys.argv) > 2 else os.path.join(os.path.dirname(os.path.dirname(
        os.path.abspath(__file__))), 'tests', 'golden'))
