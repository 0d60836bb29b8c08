"""Time the fused KITTI evaluation on a 3769-frame synthetic val set (KITTI val's size; oracle.kitti_eval.synthetic_annos,
Car / Pedestrian / Cyclist, AOS on): the device time of vc_kitti_eval (CUDA events) and the host wall time of
kitti_eval.get_official_eval_result, packing, upload, read-back and the string included.  With --reference ROOT (a
machine with the reference's sources and numba) it also times, on the host cores, the reference's own
get_official_eval_result with its rotated-box kernel under numba's CUDA simulator, and with --oracle the numpy
restatement.  Prints one JSON line.

    python profiles/microbench_kitti_eval.py [--frames 3769] [--reps 10] [--reference ROOT] [--oracle]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np   # noqa: E402

from oracle import kitti_eval as K   # noqa: E402


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:       # noqa: BLE001
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=3769)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--reference', default=None)
    ap.add_argument('--oracle', action='store_true')
    a = ap.parse_args()
    g, d = K.synthetic_annos(7, a.frames, check_near=False)
    classes = [0, 1, 2]
    res = {'frames': a.frames, 'gt': sum(len(x['name']) for x in g), 'dt': sum(len(x['name']) for x in d),
           'host_cores': os.cpu_count()}
    if a.reference:
        os.environ['NUMBA_ENABLE_CUDASIM'] = '1'
        from virconv_b200 import reference_env
        reference_env.install(reference_root=a.reference)
        import importlib
        ev = importlib.import_module('pcdet.datasets.kitti.kitti_object_eval_python.eval')
        t = time.perf_counter()
        ev.get_official_eval_result(g, d, classes)
        res['reference_cudasim_s'] = time.perf_counter() - t
    if a.oracle:
        from virconv_b200 import kitti_eval as ke
        t = time.perf_counter()
        K.evaluate(g, d, classes, ke._OFFICIAL_MIN_OVERLAPS[:, :, classes], True)
        res['oracle_s'] = time.perf_counter() - t
    import torch
    if torch.cuda.is_available():
        from virconv_b200 import _lib, ops
        from virconv_b200 import kitti_eval as ke
        res['gpu'] = gpu_info()
        mo = ke._OFFICIAL_MIN_OVERLAPS[:, :, classes]
        ke.get_official_eval_result(g, d, classes)          # warm-up: module load, allocator
        gt, dt, offs, P = ke.pack(g, d)
        F, NG, ND, C, Kk = offs.shape[1] - 1, len(gt), len(dt), 3, 2
        lane_mo = np.array([mo[k, m, c] for m in range(3) for c in range(C) for dd in range(3) for k in range(Kk)])
        dev = torch.device('cuda', 0)
        buf, (p_gt, p_dt, p_offs, p_mo) = ke._upload([gt, dt, offs, lane_mo], dev)
        ov = torch.empty(3 * P, dtype=torch.float64, device=dev)
        out = torch.empty(3 * C * 3 * Kk * ke.LANE_W, dtype=torch.float64, device=dev)
        lib = _lib.load()
        wsb = lib.vc_kitti_eval_ws_bytes(F, NG, ND, C, Kk)
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        cls = _lib.host_i32(classes)
        dev_ms = []
        for _ in range(a.reps + 2):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(lib.vc_kitti_eval(p_gt, p_dt, p_offs, p_mo, F, NG, ND, P, C, cls, Kk, 1, ov.data_ptr(),
                                         out.data_ptr(), ws.data_ptr(), wsb, ops._stream()), 'vc_kitti_eval')
            e1.record()
            torch.cuda.synchronize()
            dev_ms.append(e0.elapsed_time(e1))
        dev_ms = sorted(dev_ms[2:])
        host_ms = []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t = time.perf_counter()
            ke.get_official_eval_result(g, d, classes)
            host_ms.append(1e3 * (time.perf_counter() - t))
        host_ms.sort()
        res.update(device_ms_median=dev_ms[len(dev_ms) // 2], device_ms_min=dev_ms[0], device_ms_max=dev_ms[-1],
                   host_ms_median=host_ms[len(host_ms) // 2], host_ms_min=host_ms[0], host_ms_max=host_ms[-1])
        t0 = time.perf_counter()
        ke.pack(g, d)
        res['pack_ms'] = 1e3 * (time.perf_counter() - t0)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
