"""GPU tests of the StVD input front end inside the captured step (graph.GraphedStep / GraphedForward with the voxeliser's
`input_discard` entry): the batch carries the collated, un-split cloud, and the replay's front end + voxelisers + step equal
the eager front end run with the replay's seed followed by an exact step; replays draw afresh; ROT_NUM copies draw
independently."""
import pytest
import torch

from oracle.testing import fill_module, rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
PC = (0, -40, -3, 70.4, 40, 1)
MAX_VOXELS = 3000


def _vox(later_fusion):
    return dict(point_cloud_range=PC, voxel_size=(0.05, 0.05, 0.05), max_points_per_voxel=5, max_voxels=MAX_VOXELS,
                vfe_model='max', max_voxels_mm=MAX_VOXELS, vfe_model_mm=None,
                input_discard=dict(rate=0.8, later_fusion=later_fusion))


def _raw_batch(ids, training=True, rot=1):
    """The collated un-split cloud of each copy (indicator 2 LiDAR, 1 virtual), as collate_batch builds it before the split."""
    from virconv_b200 import scenes
    pb = scenes.make_points_batch(ids, training=training, n_lidar=4096, n_virtual=12000)
    bd = {'batch_size': pb.batch_size, 'calib': pb.calib}
    for r in range(rot):
        bd['points' + (str(r) if r else '')] = torch.from_numpy(pb.points).to(DEV)
    if training:
        bd['aug_param'] = torch.from_numpy(pb.aug_param)
    return bd


def _named(out, groups):
    named = {f'{g}:{k}': t for g in groups for k, t in out[g].items()}
    named['out'] = out['encoded_spconv_tensor']
    return named


def _eager_reference(model, batch, seed, later_fusion, loss_fn):
    """The eager front end with the replay's seed, the voxelisers, one exact step -> (loss, grads, voxel coords)."""
    from virconv_b200 import ops, preprocess
    for p in model.parameters():
        p.grad = None
    r = preprocess.input_front_end(batch['points'], batch['batch_size'], model.training, later_fusion, seed=seed,
                                   point_cloud_range=PC)
    bd = dict(batch)
    vox = {}
    for s, vfe in (('', 'max'), ('_mm', None)):
        if 'points' + s not in r:
            continue
        f, c, _ = ops.voxelize_mean(r['points' + s], batch['batch_size'], PC, (0.05, 0.05, 0.05), 5, MAX_VOXELS, vfe)
        bd.update({'voxel_features' + s: f, 'voxel_coords' + s: c.float()})
        vox[s] = c
    bd.pop('points', None)
    loss = loss_fn(model(bd))
    loss.backward()
    torch.cuda.synchronize()
    return float(loss), {k: p.grad.clone() for k, p in model.named_parameters()}, vox


def _grad_close(got, ref):
    got, ref = got.double().cpu(), ref.double().cpu()
    return float((got - ref).norm() / ref.norm().clamp_min(1e-30)) < 1e-2 and rel_err(got.float(), ref.float()) < 3e-2


@pytest.mark.parametrize('variant', ['T', 'L'])
def test_graphed_step_matches_eager_front_end(lib_built, variant):
    from virconv_b200.backbone import VirConv8x, VirConvL8x
    from virconv_b200.graph import GraphedStep, masked_mean
    later_fusion = variant == 'T'
    if later_fusion:
        model = VirConv8x(dict(CFG, LAYER_DISCARD_RATE=0.15, MM=True), 8, [1408, 1600, 80], precision='bf16')
        groups = ('multi_scale_3d_features', 'multi_scale_3d_features_mm')
        fill_module(model, 667)
    else:
        model = VirConvL8x(CFG, 8, [1408, 1600, 80], precision='bf16')
        groups = ('multi_scale_3d_features',)
        fill_module(model, 666)
    model = model.to(DEV).train()

    def loss_fn(out):
        return sum(masked_mean(t) for t in _named(out, groups).values())
    step = GraphedStep(model, loss_fn, margin=1.35, grain=256, voxelizer=_vox(later_fusion))
    batch = _raw_batch([41, 42])
    seeds, graph_grads = [], None
    for _ in range(2):
        loss = float(step(batch))
        torch.cuda.synchronize()
        if graph_grads is None:                      # the graph's own gradient tensors (an eager step rebinds p.grad)
            graph_grads = {k: p.grad for k, p in model.named_parameters()}
        grads = {k: g.clone() for k, g in graph_grads.items()}
        seed = step.inputs.seed.clone()
        seeds.append(int(seed))
        l0, g0, _ = _eager_reference(model, batch, seed, later_fusion, loss_fn)
        assert abs(loss - l0) < 1e-5 * max(1.0, abs(l0))
        for k in grads:
            assert _grad_close(grads[k], g0[k]), k
    assert seeds[0] != seeds[1]                                        # a fresh draw per replay
    assert step.recaptures == 1
    assert int(step.flags.overflow[step.flags.keys.index('stvd_input')]) == 0


def test_replays_draw_different_subsets(lib_built):
    from virconv_b200.backbone import VirConv8x
    from virconv_b200.graph import GraphedStep, masked_mean
    model = VirConv8x(dict(CFG, LAYER_DISCARD_RATE=0.15, MM=True), 8, [1408, 1600, 80], precision='bf16')
    fill_module(model, 667)
    model = model.to(DEV).train()
    groups = ('multi_scale_3d_features', 'multi_scale_3d_features_mm')
    holder = {}

    def loss_fn(out):
        holder['kept'] = out['stvd_input_kept_mm']
        return sum(masked_mean(t) for t in _named(out, groups).values())
    step = GraphedStep(model, loss_fn, margin=1.35, grain=256, voxelizer=_vox(True))
    batch = _raw_batch([43, 44])
    subsets = []
    for _ in range(2):
        step(batch)
        torch.cuda.synchronize()
        k = holder['kept']
        subsets.append(k[:int(k.num_rows)].sort().values.cpu())
    assert not torch.equal(subsets[0], subsets[1])


def test_pipelined_step_refuses_the_front_end(lib_built):
    from virconv_b200.backbone import VirConvL8x
    from virconv_b200.graph import PipelinedStep
    model = VirConvL8x(CFG, 8, [1408, 1600, 80]).to(DEV).train()
    with pytest.raises(ValueError):
        PipelinedStep(model, lambda out: None, voxelizer=_vox(False))


def test_graphed_forward_rot3_copies_draw_independently(lib_built):
    """ROT_NUM = 3 copies of the same cloud, eval: each copy's front end draws its own subset (bin_num 10, no shuffle), and
    the captured forward equals the eager eval forward fed the eager front end of every copy under the replay's seed."""
    from virconv_b200 import ops, preprocess
    from virconv_b200.backbone import VirConv8x
    from virconv_b200.graph import GraphedForward
    model = VirConv8x(dict(CFG, LAYER_DISCARD_RATE=0.15, MM=True), 8, [1408, 1600, 80], precision='bf16')
    fill_module(model, 667)
    model = model.to(DEV).eval()
    batch = _raw_batch([45, 46], training=False, rot=3)
    from virconv_b200 import scenes
    batch['transform_param'] = torch.from_numpy(scenes.TEST_TRANSFORMS[None].repeat(2, 0).copy())
    fwd = GraphedForward(model, voxelizer=_vox(True))
    out = fwd(batch)
    torch.cuda.synchronize()
    seed = fwd.inputs.seed.clone()
    kept = [out['stvd_input_kept_mm' + s] for s in ('', '1', '2')]
    kept = [k[:int(k.num_rows)].cpu() for k in kept]
    assert not torch.equal(kept[0], kept[1]) and not torch.equal(kept[1], kept[2])
    bd = dict(batch)
    for i, s in enumerate(('', '1', '2')):
        r = preprocess.input_front_end(batch['points' + s], 2, False, True, seed=seed, draw=i, point_cloud_range=PC)
        assert torch.equal(r['stvd_input_kept_mm'].cpu(), kept[i])
        for key, vfe in (('', 'max'), ('_mm', None)):
            f, c, _ = ops.voxelize_mean(r['points' + key], 2, PC, (0.05, 0.05, 0.05), 5, MAX_VOXELS, vfe)
            bd.update({'voxel_features' + key + s: f, 'voxel_coords' + key + s: c.float()})
        bd.pop('points' + s)
    with torch.no_grad():
        ref = model(bd)
    for s in ('', '1', '2'):
        t, e = out['encoded_spconv_tensor' + s], ref['encoded_spconv_tensor' + s]
        rows = int(t.num_rows)
        assert rows == e.features.shape[0], s
        assert torch.equal(t.indices[:rows].int(), e.indices.int()), s
        assert rel_err(t.features[:rows].float().cpu(), e.features.float().cpu()) < 1e-2, s
