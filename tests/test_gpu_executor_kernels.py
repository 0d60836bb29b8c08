"""GPU test of which conv launches the plan executor picks for every layer of a VirConvL8x step: forward, weight gradient
and input gradient, in each precision / BatchNorm mode a training or fine-tuning step uses."""
import pytest
import torch

from oracle.testing import fill_module

pytestmark = pytest.mark.gpu
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
N_LAYERS = 20                                      # plan order: 0-3 block 1, 4-8 block 2, 9-13 block 3, 14-18 block 4, 19 conv_out
IMAGE_C8 = (2, 3)                                  # image-branch (2-D) layers of block 1: C = 8
IMAGE = (7, 8, 12, 13, 17, 18)                     # the other image-branch layers


def _expected(fwd, wgrad, dgrad_c8, dgrad_image, dgrad_rest):
    out = {}
    for li in range(N_LAYERS):
        dgrad = [] if li == 0 else [dgrad_c8 if li in IMAGE_C8 else dgrad_image if li in IMAGE else dgrad_rest]
        out[li] = sorted([fwd, wgrad] + dgrad)
    return out


@pytest.mark.parametrize('precision,bn_training,want', [
    ('bf16', True, _expected('conv_fwd_tc', 'conv_wgrad_tc', 'conv_dgrad_scatter', 'conv_dgrad_scatter_tc', 'conv_dgrad_tc')),
    ('bf16', False, _expected('conv_fwd_tc', 'conv_wgrad', 'conv_dgrad_scatter', 'conv_dgrad_scatter', 'conv_dgrad')),
    ('fp32', True, _expected('conv_fwd', 'conv_wgrad', 'conv_dgrad_scatter', 'conv_dgrad_scatter', 'conv_dgrad')),
])
def test_plan_step_kernel_per_layer(precision, bn_training, want):
    """One eager step (forward + backward) between executor.timing_start() and timing_stop(): every layer runs exactly the
    forward, weight-gradient and input-gradient launches of the table, and layer 0 (the network input) no input gradient."""
    from virconv_b200 import executor, scenes
    from virconv_b200.backbone import VirConvL8x
    from virconv_b200.graph import masked_mean
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], precision=precision)
    fill_module(m, 666)
    m = m.cuda().train(bn_training)
    b = scenes.make_batch([3, 4], n_lidar=4096, n_virtual=9000, max_voxels=7000, training=True)
    bd = {'voxel_features': torch.from_numpy(b.voxel_features.copy()).cuda(),
          'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).cuda(), 'batch_size': b.batch_size, 'calib': b.calib,
          'aug_param': torch.from_numpy(b.aug_param.copy())}
    assert len(m._plan().layers) == N_LAYERS
    executor.timing_start()
    try:
        out = m(dict(bd))
        loss = sum(masked_mean(t) for t in list(out['multi_scale_3d_features'].values()) + [out['encoded_spconv_tensor']])
        loss.backward()
    finally:
        recs = executor.timing_stop()
    got = {li: [] for li in range(N_LAYERS)}
    for kind, layer, _ in recs:
        got[layer].append(kind)
    assert {li: sorted(k) for li, k in got.items()} == want
