"""Record tests/golden/stvd_input_plan.npz from the reference's own `DatasetTemplate.partition` / `input_point_discard`
(pcdet/datasets/dataset.py:120-189) — TEST INFRASTRUCTURE, runs on the CPU where the reference sources are, in the pattern
of oracle/make_golden.py.  What it pins does not depend on the random draw: per case, the reference's `position`, its
`distant_points_num_acc`, the size of every part (far -> near) before and after the discard, and whether it raised
ZeroDivisionError.

usage:  python -m oracle.stvd_input_golden
"""
from __future__ import annotations

import os

import numpy as np

from .make_golden import OUT, import_reference, import_reference_dataset


def cases():
    """(name, points [N, 1] float32 (x: the only column the discard reads), bin_num, rate): the edge cases of the plan at
    bin_num 2 and 10."""
    rng = np.random.default_rng(2024)

    def cloud(xs):
        return np.asarray(xs, np.float32).reshape(-1, 1)
    out = []
    for bn in (2, 10):
        out += [
            (f'uniform_b{bn}', cloud(rng.uniform(0, 70, 2000)), bn, 0.8),
            (f'near_heavy_b{bn}', cloud(np.abs(rng.normal(0, 8, 3000))), bn, 0.8),
            (f'one_bin_near_b{bn}', cloud(rng.uniform(0, 2, 1500)), bn, 0.8),            # every point in bin 0
            (f'one_bin_far_b{bn}', cloud(rng.uniform(61, 80, 1500)), bn, 0.8),           # every point in the open last bin
            (f'empty_bins_b{bn}', cloud(np.r_[rng.uniform(0, 3, 900), rng.uniform(50, 59, 100)]), bn, 0.8),
            (f'neg_nan_b{bn}', cloud(np.r_[rng.uniform(-20, 70, 2000), [np.nan] * 40]), bn, 0.8),
            (f'mostly_dropped_b{bn}', cloud(np.r_[rng.uniform(-30, -1, 1500), rng.uniform(0, 60, 200)]), bn, 0.8),
            (f'rate05_b{bn}', cloud(rng.uniform(0, 70, 2000)), bn, 0.5),
            (f'rate0_b{bn}', cloud(rng.uniform(0, 70, 1000)), bn, 0.0),
            (f'tiny_b{bn}', cloud(rng.uniform(0, 60, 3)), bn, 0.8),
            (f'single_b{bn}', cloud([5.0]), bn, 0.8),
            (f'empty_b{bn}', cloud([]), bn, 0.8),                                          # a scene without virtual points
        ]
    return out


def main():
    import_reference()                       # (the pcdet package stubs)
    ds_mod = import_reference_dataset()
    ds = ds_mod.DatasetTemplate.__new__(ds_mod.DatasetTemplate)
    part = ds.partition
    res, lines = {}, []
    for name, pts, bn, rate in cases():
        seen = {}

        def spy(*a, **k):
            seen['r'] = part(*a, **k)
            seen['before'] = [p.shape[0] for p in seen['r'][0]]
            return seen['r']
        ds.partition = spy
        np.random.seed(0)
        try:
            ds.input_point_discard(pts.copy(), bin_num=bn, rate=rate)
            parts, position, distant = seen['r']
            after = [p.shape[0] for p in parts]
            zero_div = 0
        except ZeroDivisionError:
            position, distant, zero_div = -1, -1, 1
            after = [0] * bn
            seen['before'] = [0] * bn
        res[f'{name}:points'] = pts
        res[f'{name}:meta'] = np.array([bn, position, distant, zero_div], np.int64)
        res[f'{name}:rate'] = np.float64(rate)
        res[f'{name}:before'] = np.array(seen['before'], np.int64)
        res[f'{name}:after'] = np.array(after, np.int64)
        lines.append(f'{name}: N={pts.shape[0]} bins={bn} rate={rate} position={position} distant={distant} '
                     f'parts {seen["before"]} -> {after} zero_div={zero_div}')
    ds.partition = part
    np.savez_compressed(os.path.join(OUT, 'stvd_input_plan.npz'), names=np.array([c[0] for c in cases()]), **res)
    print('\n'.join(lines))


if __name__ == '__main__':
    main()
