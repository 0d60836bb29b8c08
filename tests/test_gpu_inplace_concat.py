"""GPU tests of the bf16 plan step's concat written in place, the fp32 copies it no longer writes, and the two-kernel
masked_mean loss helper."""
import numpy as np
import pytest
import torch

from oracle.testing import fill_module

pytestmark = pytest.mark.gpu
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])


def _features(cap, c, n, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(cap, c, generator=g) * 3 + 0.5
    x[n:] = 0
    return x.cuda()


@pytest.mark.parametrize('cap,c,n', [(1000, 16, 777), (5000, 64, 5000), (300, 32, 0), (123457, 64, 100003)])
def test_masked_mean_static(cap, c, n):
    from virconv_b200.graph import _MaskedMean
    x = _features(cap, c, n, cap).requires_grad_(True)
    nd = torch.tensor([n], dtype=torch.int32, device='cuda')
    m = _MaskedMean.apply(x, nd)
    m2 = _MaskedMean.apply(x, nd)
    assert m.item() == m2.item() or (n == 0 and np.isnan(m.item()) and np.isnan(m2.item()))   # deterministic
    if n > 0:
        want = x[:n].double().mean().item()
        assert abs(m.item() - want) <= 1e-6 * max(abs(want), 1e-6)
        (3.0 * m).backward()
        g = x.grad
        assert g.is_contiguous() and g.shape == x.shape
        want_g = torch.full_like(g[:n], 3.0 / (n * c))
        assert torch.allclose(g[:n], want_g, rtol=1e-6, atol=0) and torch.all(g[n:] == 0)


def test_masked_mean_exact():
    from virconv_b200.graph import masked_mean

    class T:
        pass
    t = T()
    t.features = _features(4097, 32, 4097, 7).requires_grad_(True)
    m = masked_mean(t)
    want = t.features.double().mean().item()
    assert abs(m.item() - want) <= 1e-6 * abs(want)
    assert masked_mean(t).item() == m.item()
    m.backward()
    assert torch.allclose(t.features.grad, torch.full_like(t.features, 1.0 / t.features.numel()), rtol=1e-6, atol=0)


def test_plan_step_launches_no_concat_kernel():
    """bf16 training step through the plan executor: the BN-apply of the two input layers of every NRConv block writes its
    column slice of the concat, and the backward hands each input its column slice of the concat's gradient (the image
    branch's scatter dgrad adds into the first one in place), so no concat kernel runs in either direction.  Both halves of
    the fp32 concat and of its bf16 shadow are written, and the gradients match the exact fp32-copy route within the bf16
    mode's run-to-run noise (checked by test_gpu_graph.py and smoke(); here: finite and non-zero)."""
    from torch.profiler import ProfilerActivity, profile
    from virconv_b200 import scenes
    from virconv_b200.backbone import VirConvL8x
    from virconv_b200.graph import masked_mean
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], precision='bf16')
    fill_module(m, 666)
    m = m.cuda().train()
    b = scenes.make_batch([3, 4], n_lidar=4096, n_virtual=9000, max_voxels=7000, training=True)
    bd = {'voxel_features': torch.from_numpy(b.voxel_features.copy()).cuda(),
          'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).cuda(), 'batch_size': b.batch_size, 'calib': b.calib,
          'aug_param': torch.from_numpy(b.aug_param.copy())}

    def step():
        for p in m.parameters():
            p.grad = None
        out = m(dict(bd))
        loss = sum(masked_mean(t) for t in list(out['multi_scale_3d_features'].values()) + [out['encoded_spconv_tensor']])
        loss.backward()
        torch.cuda.synchronize()
        return out

    step()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = step()
    names = [e.name() for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA]
    assert any('tc_scatter_kernel' in n for n in names)
    assert not any('cat2' in n for n in names), 'a concat kernel ran'
    for k, t in out['multi_scale_3d_features'].items():
        fb = t.features_bf16
        assert fb is not None and fb.shape == t.features.shape, k
        assert torch.equal(fb, t.features.to(torch.bfloat16)), k        # both column halves written, bf16 of the fp32 values
    for name, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().max() > 0, name
