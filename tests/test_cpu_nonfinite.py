"""The float64 / numpy references tests/test_gpu_nonfinite.py holds the kernels to, on non-finite and boundary values: they
must treat NaN and Inf as torch and the reference's data pipeline do, or the GPU comparisons would check nothing."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import audit
from virconv_b200 import scenes

NAN, INF = float('nan'), float('inf')
RANGE = (0, -40, -3, 70.4, 40, 1)


def test_relu_and_its_backward_pass_nan():
    x = torch.tensor([NAN, -1.0, 2.0, -0.0, INF, -INF], dtype=torch.float64, requires_grad=True)
    y = torch.relu(x)
    assert torch.isnan(y[0]) and y[4] == INF and y[5] == 0
    y.backward(torch.full_like(x, 3.0))
    assert x.grad.tolist() == [3.0, 0.0, 3.0, 0.0, 3.0, 0.0]      # threshold_backward: passes unless the output is <= 0
    m = audit.relu_mask(x.detach(), torch.zeros(1), torch.ones(1), torch.ones(1), torch.zeros(1))
    assert not m[0]                                                 # (why the GPU tests take backward refs from autograd)


def test_batch_norm_nan_and_inf_channels():
    x = torch.randn(40, 4, dtype=torch.float64)
    x[3, 1], x[5, 2], x[7, 3] = NAN, INF, -INF
    rm, rv = torch.zeros(4, dtype=torch.float64), torch.ones(4, dtype=torch.float64)
    y = torch.relu(F.batch_norm(x, rm, rv, torch.ones(4, dtype=torch.float64), torch.zeros(4, dtype=torch.float64), True, 0.01, 1e-3))
    assert torch.isfinite(y[:, 0]).all() and not torch.isfinite(y[:, 1:]).any()
    assert torch.isfinite(rm[0]) and not torch.isfinite(rm[1:]).any() and not torch.isfinite(rv[1:]).any()
    mean, invstd, _, _ = audit.batch_stats(x, 1e-3)
    assert torch.isfinite(mean[0]) and not torch.isfinite(invstd[1:]).any()


def test_max_pool_propagates_nan():
    v = torch.tensor([[[[1.0, NAN, 3.0, NAN, 0.5]]]], dtype=torch.float64)
    out, idx = F.max_pool2d(v, kernel_size=[1, 5], return_indices=True)
    assert torch.isnan(out).all() and int(idx) in (1, 3)


def test_voxeliser_reference_drops_nonfinite_and_out_of_range_points():
    p = np.array([[10.0, 0.0, -1.0, 0.5],
                  [NAN, 0.0, -1.0, 0.5], [10.0, NAN, -1.0, 0.5], [10.0, 0.0, NAN, 0.5],
                  [INF, 0.0, -1.0, 0.5], [10.0, -INF, -1.0, 0.5], [10.0, 0.0, INF, 0.5],
                  [0.0, -40.0, -3.0, 0.5],                                              # on the lower bound: kept
                  [70.4, 0.0, -1.0, 0.5], [20.0, 40.0, -1.0, 0.5],                      # on the upper bound: dropped
                  [np.nextafter(np.float32(70.4), np.float32(0)), 0.0, -1.0, 0.5],       # one ulp below: kept
                  [30.0, 0.0, -1.0, NAN]], np.float32)
    with np.errstate(invalid='ignore'):
        vox, coords, num = scenes.voxelize_first_come(scenes.mask_points_by_range(p, RANGE), pc_range=RANGE)
    assert coords.tolist() == [[40, 800, 200], [0, 0, 0], [40, 800, 1407], [40, 800, 600]]
    f = scenes.mean_vfe(vox, num, 'max')
    assert np.isnan(f[3, 3]) and np.isfinite(f[:3]).all()
