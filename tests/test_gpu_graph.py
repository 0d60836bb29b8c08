"""GPU tests of the configuration bench.py measures: bf16 tensor-core kernels + plan executor in STATIC mode (device
row counts, capacity-sized buffers) + whole-step CUDA graph replay over rotating batches, against the exact-shape,
host-synchronised execution of the same step (which the other test files pin against the oracle)."""
import numpy as np
import pytest
import torch

from oracle.testing import fill_module, rel_err

pytestmark = pytest.mark.gpu
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
KEYS = ('x_conv1', 'x_conv2', 'x_conv3', 'x_conv4', 'out')


def _model(precision):
    from virconv_b200.backbone import VirConvL8x
    m = VirConvL8x(CFG, 8, [1408, 1600, 80], precision=precision)
    fill_module(m, 666)
    return m.to('cuda:0').train()


def _batch(ids, n_lidar=4096, n_virtual=9000, max_voxels=7000):
    from virconv_b200 import scenes
    b = scenes.make_batch(ids, n_lidar=n_lidar, n_virtual=n_virtual, max_voxels=max_voxels, training=True)
    return {'voxel_features': torch.from_numpy(b.voxel_features.copy()).cuda(),
            'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).cuda(), 'batch_size': b.batch_size, 'calib': b.calib,
            'aug_param': torch.from_numpy(b.aug_param.copy())}


def _named(out):
    named = dict(out['multi_scale_3d_features'])
    named['out'] = out['encoded_spconv_tensor']
    return named


def _loss(out):
    from virconv_b200.graph import masked_mean
    return sum(masked_mean(t) for t in _named(out).values())


def _exact(model, batch):
    for p in model.parameters():
        p.grad = None
    out = model(dict(batch))
    loss = _loss(out)
    loss.backward()
    torch.cuda.synchronize()
    return float(loss), {k: v.grad.clone() for k, v in model.named_parameters()}, _named(out)


def _grad_close(got, ref):
    """bf16 mode: the fp32 atomics of the scatter dgrads / weight-gradient reductions land in a different order every run, and
    the bf16 rounding of the gradients they feed amplifies that — two exact-mode runs of the SAME batch already differ by a
    few 1e-3 of the largest element.  So: relative L2 error below 1e-2, largest element
    difference below 3e-2 of the largest element."""
    got, ref = got.double().cpu(), ref.double().cpu()
    l2 = float((got - ref).norm() / ref.norm().clamp_min(1e-30))
    return l2 < 1e-2 and rel_err(got.float(), ref.float()) < 3e-2


def _err_flag():
    from virconv_b200 import ops
    return int(ops.tc_error_flag(torch.device('cuda:0')).item())


@pytest.mark.parametrize('precision', ['bf16', 'fp32'])
def test_static_mode_matches_exact_mode(lib_built, precision):
    """Same batch, same weights: the static (capacity + device count) execution publishes the exact mode's tensors on
    the valid rows, zero / -1 tails beyond them, the same row counts, loss and parameter gradients."""
    from virconv_b200 import executor, ops
    model = _model(precision)
    batch = _batch([11, 12])
    l0, g0, n0 = _exact(model, batch)
    run = executor.last_run(model)
    caps = executor.measured_caps(run, 1.3, 256)
    n = batch['voxel_features'].shape[0]
    cap0 = (int(n * 1.25) + 255) // 256 * 256
    dev = torch.device('cuda:0')
    vf = torch.zeros((cap0, 8), device=dev)
    vc = torch.full((cap0, 4), -1.0, device=dev)
    vf[:n] = batch['voxel_features']
    vc[:n] = batch['voxel_coords']
    vf[n:] = float('nan')                 # whatever is beyond the count must never be read into a result
    spec = executor.StaticSpec(torch.tensor([n], dtype=torch.int32, device=dev), caps,
                               torch.zeros(1, dtype=torch.int32, device=dev))
    proj = ops.projection_params(batch['calib'], batch['aug_param'], 2, dev)
    for p in model.parameters():
        p.grad = None
    bd = {'voxel_features': vf, 'voxel_coords': vc, 'batch_size': 2, 'calib': batch['calib'], 'aug_param': batch['aug_param'],
          'virconv_static': spec, 'virconv_proj': proj}
    out = model(bd)
    loss = _loss(out)
    loss.backward()
    torch.cuda.synchronize()
    assert _err_flag() == 0
    assert int(spec.overflow.item()) == 0
    named = _named(out)
    for k in KEYS:
        t, e = named[k], n0[k]
        rows = int(t.num_rows.item())
        assert rows == e.features.shape[0], k
        assert t.features.shape[0] >= rows and t.features.shape[0] % 256 == 0, k
        assert torch.equal(t.indices[:rows].int(), e.indices.int()), k
        assert rel_err(t.features[:rows].detach().cpu(), e.features.detach().cpu()) < 1e-5, k
        assert float(t.features[rows:].abs().max()) == 0.0 if t.features.shape[0] > rows else True, k
        if k != 'x_conv1':
            assert bool((t.indices[rows:] == -1).all()), k
    assert abs(float(loss) - l0) < 1e-5 * max(1.0, abs(l0))
    for name, p in model.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), name
        if precision == 'bf16':
            assert _grad_close(p.grad, g0[name]), name
        else:
            assert rel_err(p.grad.cpu(), g0[name].cpu()) < 2e-4, name     # order of the scatter / float64 atomics differs run to run


def test_static_mode_reports_overflow(lib_built):
    from virconv_b200 import executor, ops
    model = _model('bf16')
    batch = _batch([11, 12])
    _exact(model, batch)
    caps = executor.measured_caps(executor.last_run(model), 1.0, 1)
    k = sorted(caps)[0]
    true_rows = caps[k]
    caps[k] = caps[k] - 300                # one strided conv's output set does not fit
    n = batch['voxel_features'].shape[0]
    dev = torch.device('cuda:0')
    spec = executor.StaticSpec(torch.tensor([n], dtype=torch.int32, device=dev), caps, torch.zeros(1, dtype=torch.int32, device=dev))
    bd = dict(batch)
    bd.update(virconv_static=spec, virconv_proj=ops.projection_params(batch['calib'], batch['aug_param'], 2, dev))
    with torch.no_grad():
        out = model(bd)
    torch.cuda.synchronize()
    assert int(spec.overflow.item()) == true_rows          # the row count that did not fit
    assert bool(torch.isfinite(out['encoded_spconv_tensor'].features).all())


def test_graph_replay_matches_eager_over_rotating_batches(lib_built):
    """What bench.py times: >= 8 back-to-back replays of the captured step (bf16, wgrad stream, index stream, no host
    synchronisation between steps) over rotating batches; every step's loss and parameter gradients against a
    synchronous exact-mode execution of the same batch with the same weights."""
    from virconv_b200.graph import GraphedStep
    model = _model('bf16')
    batches = [_batch([20 + 2 * i, 21 + 2 * i]) for i in range(4)]
    ref = []
    for b in batches:
        l, g, _ = _exact(model, b)
        ref.append((l, g))
    step = GraphedStep(model, _loss, margin=1.35, grain=256)
    params = dict(model.named_parameters())
    losses, grads = [], []
    for s in range(9):
        loss = step(batches[s % 4])
        losses.append(loss.detach().clone())                       # device-side copies, no synchronisation
        grads.append({k: v.grad.detach().clone() for k, v in params.items()})
    torch.cuda.synchronize()
    assert _err_flag() == 0
    assert step.recaptures == 1
    for s in range(9):
        l0, g0 = ref[s % 4]
        assert abs(float(losses[s]) - l0) < 1e-5 * max(1.0, abs(l0)), s
        for k in params:
            assert _grad_close(grads[s][k], g0[k]), (s, k)


def test_graph_recaptures_when_a_batch_does_not_fit(lib_built):
    from virconv_b200.graph import GraphedStep
    model = _model('bf16')
    small = _batch([31, 32], n_lidar=2048, n_virtual=3000, max_voxels=2500)
    big = _batch([33, 34], n_lidar=4096, n_virtual=9000, max_voxels=7000)
    step = GraphedStep(model, _loss, margin=1.05, grain=64)
    step(small)
    torch.cuda.synchronize()
    assert step.recaptures == 1
    l_big, g_big, _ = _exact(model, big)
    loss = step(big)                                                # more input rows than the buffers hold -> re-capture
    torch.cuda.synchronize()
    assert step.recaptures == 2
    assert abs(float(loss) - l_big) < 1e-5 * max(1.0, abs(l_big))


def test_capture_outlives_unreachable_graphs_of_earlier_steps(lib_built):
    """An earlier GraphedStep dropped inside a reference cycle keeps its CUDA graphs until the cyclic collector runs, and a
    graph destroyed during another capture invalidates that capture.  The collector runs here in the middle of the capture
    (from the loss function), so it must find no such graph left."""
    import gc
    from virconv_b200.graph import GraphedStep
    model = _model('bf16')
    batch = _batch([35, 36], n_lidar=2048, n_virtual=3000, max_voxels=2500)
    old = GraphedStep(model, _loss, margin=1.3, grain=256)
    old(batch)
    torch.cuda.synchronize()
    old.cycle = old
    del old

    def loss_collecting(out):
        if torch.cuda.is_current_stream_capturing():
            gc.collect()
        return _loss(out)

    l0, _, _ = _exact(model, batch)
    step = GraphedStep(model, loss_collecting, margin=1.3, grain=256)
    loss = step(batch)
    torch.cuda.synchronize()
    assert step.recaptures == 1
    assert abs(float(loss) - l0) < 1e-5 * max(1.0, abs(l0))


def test_graph_resets_the_input_tail_of_a_shrinking_batch(lib_built):
    """A larger batch, then a smaller one through the same captured step (voxelised batches): the published x_conv1, whose
    indices are the graph's input coordinates, keeps its -1 tail past `num_rows` — no row of the larger batch is left
    behind — and loss and gradients equal the exact step's."""
    from virconv_b200.graph import GraphedStep
    model = _model('bf16')
    big = _batch([71, 72])
    small = _batch([73, 74], n_lidar=2048, n_virtual=3000, max_voxels=2500)
    l_s, g_s, _ = _exact(model, small)
    held = {}

    def loss_fn(out):
        held['x_conv1'] = out['multi_scale_3d_features']['x_conv1']
        return _loss(out)

    step = GraphedStep(model, loss_fn, margin=1.35, grain=256)
    step(big)
    loss = step(small)
    torch.cuda.synchronize()
    assert _err_flag() == 0 and step.recaptures == 1
    x1 = held['x_conv1']                                            # (the tensor of the capture: the replays rewrite it)
    rows = int(x1.num_rows.item())
    assert rows == small['voxel_features'].shape[0] < big['voxel_features'].shape[0]
    assert torch.equal(x1.indices[:rows], small['voxel_coords'].int())
    assert bool((x1.indices[rows:] == -1).all())
    assert abs(float(loss) - l_s) < 1e-5 * max(1.0, abs(l_s))
    for name, p in model.named_parameters():
        assert _grad_close(p.grad, g_s[name]), name


def test_graph_with_in_graph_voxeliser(lib_built):
    """bench.py's e2e path: raw collated points are the step's input, hash-grid voxelisation + MeanVFE run inside the
    captured graph (capacity-sized point buffer with an out-of-range tail, device voxel count); result against the exact
    execution on the host-voxelised batch of the same scenes."""
    from virconv_b200 import scenes
    from virconv_b200.graph import GraphedStep
    model = _model('bf16')
    ids = [[41, 42], [43, 44], [45, 46]]
    kw = dict(n_lidar=4096, n_virtual=9000)
    ref = []
    for i in ids:
        l, g, _ = _exact(model, _batch(i, max_voxels=7000, **kw))
        ref.append((l, g))
    vox = dict(point_cloud_range=(0, -40, -3, 70.4, 40, 1), voxel_size=(0.05, 0.05, 0.05), max_points_per_voxel=5,
               max_voxels=7000, vfe_model='max')
    step = GraphedStep(model, _loss, margin=1.35, grain=256, voxelizer=vox)
    params = dict(model.named_parameters())
    got = []
    for s in range(6):
        pb = scenes.make_points_batch(ids[s % 3], training=True, **kw)
        b = {'points': torch.from_numpy(pb.points).cuda(), 'batch_size': pb.batch_size, 'calib': pb.calib,
             'aug_param': torch.from_numpy(pb.aug_param)}
        loss = step(b)
        got.append((loss.detach().clone(), {k: v.grad.detach().clone() for k, v in params.items()}))
    torch.cuda.synchronize()
    assert _err_flag() == 0 and step.recaptures == 1
    for s in range(6):
        l0, g0 = ref[s % 3]
        assert abs(float(got[s][0]) - l0) < 1e-5 * max(1.0, abs(l0)), s
        for k in params:
            assert _grad_close(got[s][1][k], g0[k]), (s, k)


@pytest.mark.parametrize('with_voxeliser', [False, True])
def test_pipelined_step_matches_eager(lib_built, with_voxeliser):
    """graph.PipelinedStep: every step as an index graph + a feature graph over two alternating buffer sets, the index graph of
    step t+1 running beside the feature graph of step t.  Losses and parameter gradients of 8 back-to-back steps over rotating
    batches against the synchronous exact-mode execution of the same batches."""
    from virconv_b200 import scenes
    from virconv_b200.graph import PipelinedStep
    model = _model('bf16')
    ids = [[61, 62], [63, 64], [65, 66]]
    kw = dict(n_lidar=4096, n_virtual=9000)
    ref = [_exact(model, _batch(i, max_voxels=7000, **kw))[:2] for i in ids]
    vox = dict(point_cloud_range=(0, -40, -3, 70.4, 40, 1), voxel_size=(0.05, 0.05, 0.05), max_points_per_voxel=5,
               max_voxels=7000, vfe_model='max') if with_voxeliser else None
    step = PipelinedStep(model, _loss, margin=1.35, grain=256, voxelizer=vox)
    params = dict(model.named_parameters())
    got = []
    for s in range(8):
        if with_voxeliser:
            pb = scenes.make_points_batch(ids[s % 3], training=True, **kw)
            b = {'points': torch.from_numpy(pb.points).cuda(), 'batch_size': pb.batch_size, 'calib': pb.calib,
                 'aug_param': torch.from_numpy(pb.aug_param)}
        else:
            b = _batch(ids[s % 3], max_voxels=7000, **kw)
        loss = step(b)
        got.append((loss.detach().clone(), {k: v.grad.detach().clone() for k, v in params.items()}))
    torch.cuda.synchronize()
    assert _err_flag() == 0 and step.recaptures == 2          # one capture per buffer set
    for s in range(8):
        l0, g0 = ref[s % 3]
        assert abs(float(got[s][0]) - l0) < 1e-5 * max(1.0, abs(l0)), s
        for k in params:
            assert _grad_close(got[s][1][k], g0[k]), (s, k)
