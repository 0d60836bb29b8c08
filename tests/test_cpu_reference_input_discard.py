"""`reference_env.install(use_device_input_discard=True)` against the reference's own unmodified dataset code (only where
/root/reference exists): the input discard and the shuffle pass the points through, the range mask filters the boxes only."""
import functools
import os
import sys
import types

import numpy as np
import pytest

REF = '/root/reference'
pytestmark = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, 'pcdet')), reason='no /root/reference on this machine')


def test_dataset_hands_over_the_undiscarded_cloud():
    saved = dict(sys.modules)
    try:
        import virconv_b200.reference_env as renv
        renv.install(reference_root=REF, use_device_input_discard=True)
        from pcdet.datasets.dataset import DatasetTemplate
        from pcdet.datasets.processor.data_processor import DataProcessor
        from pcdet.utils import box_utils
        pts = np.random.default_rng(0).uniform(-80, 80, (500, 8)).astype(np.float32)
        assert DatasetTemplate.input_point_discard(None, pts, bin_num=2, rate=0.8) is pts
        pcr = np.array([0, -40, -3, 70.4, 40, 1], dtype=np.float32)
        dp = types.SimpleNamespace(rot_num=2, point_cloud_range=pcr, training=True, mode='train')
        dp.shuffle_points = functools.partial(DataProcessor.shuffle_points, dp)
        dp.mask_points_and_boxes_outside_range = functools.partial(DataProcessor.mask_points_and_boxes_outside_range, dp)
        cfg = types.SimpleNamespace(REMOVE_OUTSIDE_BOXES=True, SHUFFLE_ENABLED={'train': True, 'test': False},
                                    get=lambda k, d=None: d)
        boxes = np.array([[10, 0, 0, 4, 2, 1.5, 0], [-30, 0, 0, 4, 2, 1.5, 0], [60, 39, 0, 4, 2, 1.5, 0]], np.float32)
        d = {'points': pts.copy(), 'points1': pts.copy(), 'gt_boxes': boxes.copy(), 'gt_boxes1': boxes.copy()}
        out = DataProcessor.mask_points_and_boxes_outside_range(dp, dict(d), cfg)
        want = boxes[box_utils.mask_boxes_outside_range_numpy(boxes, pcr, min_num_corners=1)]
        assert 0 < want.shape[0] < boxes.shape[0]
        for s in ('', '1'):
            assert np.array_equal(out['points' + s], pts)
            assert np.array_equal(out['gt_boxes' + s], want)
        out = DataProcessor.shuffle_points(dp, dict(d), cfg)
        assert np.array_equal(out['points'], pts)
    finally:
        for k in list(sys.modules):
            if k not in saved and k.split('.')[0] in ('pcdet', 'spconv', 'cumm', 'easydict', 'tensorboardX',
                                                      'prefetch_generator', 'skimage', 'train_utils'):
                del sys.modules[k]
