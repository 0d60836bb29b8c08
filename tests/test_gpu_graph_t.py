"""GPU tests of the VirConv-T / VirConv-S training step in static mode and under graph.GraphedStep: VirConv8x's LiDAR stream
and virtual-point (MM) stream, each with its own StaticSpec, input buffers and overflow flag, against the exact-shape,
host-synchronised execution of the same step (which tests/test_gpu_backbone.py pins against the oracle)."""
import copy

import numpy as np
import pytest
import torch

from oracle import rulebook as orb
from oracle.testing import fill_module, rel_err

pytestmark = pytest.mark.gpu
CFG8 = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.15, NUM_FILTERS=[16, 32, 64, 64], MM=True)
DEV = torch.device('cuda:0')
GROUPS = ('multi_scale_3d_features', 'multi_scale_3d_features_mm')
STREAMS = ('', '_mm')
KW = dict(n_lidar=4096, n_virtual=6000)
MAX_VOXELS = 3000


@pytest.fixture(autouse=True)
def _no_pipeline_timeout(lib_built):
    """Every test leaves the tensor-core kernels' pipeline-timeout flag at 0."""
    yield
    from virconv_b200 import ops
    torch.cuda.synchronize()
    assert int(ops.tc_error_flag(DEV).item()) == 0


def _model(precision='bf16', **kw):
    from virconv_b200.backbone import VirConv8x
    m = VirConv8x(CFG8, 8, [1408, 1600, 80], precision=precision, **kw)
    fill_module(m, 667)
    return m.to(DEV).train()


def _batch(ids, max_voxels=MAX_VOXELS, **kw):
    from virconv_b200 import scenes
    b = scenes.make_batch_mm(ids, max_voxels=max_voxels, training=True, **dict(KW, **kw))
    bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
    bd.update(batch_size=b.batch_size, calib=b.calib, aug_param=torch.from_numpy(b.aug_param.copy()))
    return bd


def _points_batch(ids):
    """The collated points of the same scenes, split into the two streams by the indicator column (2 = LiDAR, 1 = virtual)."""
    from virconv_b200 import scenes
    pb = scenes.make_points_batch(ids, training=True, **KW)
    p = torch.from_numpy(pb.points)
    return {'points': p[p[:, 8] == 2].contiguous().to(DEV), 'points_mm': p[p[:, 8] == 1].contiguous().to(DEV),
            'batch_size': pb.batch_size, 'calib': pb.calib, 'aug_param': torch.from_numpy(pb.aug_param)}


def _named(out):
    named = {f'{g}:{k}': t for g in GROUPS for k, t in out[g].items()}
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
    return float(loss.detach()), {k: v.grad.clone() for k, v in model.named_parameters()}, _named(out)


def _grad_close(got, ref):
    """The bf16 criterion of test_gpu_graph.py: relative L2 below 1e-2, largest difference below 3e-2 of the largest element."""
    got, ref = got.double().cpu(), ref.double().cpu()
    return float((got - ref).norm() / ref.norm().clamp_min(1e-30)) < 1e-2 and rel_err(got.float(), ref.float()) < 3e-2


def _static_batch(batch, caps, cap_margin=1.25, grain=256, tail=float('nan')):
    """The batch in static form: per stream capacity-sized inputs (rows past the count filled with `tail`, -1 coordinates),
    the device row count and its own overflow flag; the shared projection block on the device."""
    from virconv_b200 import executor, ops
    bd = {'batch_size': batch['batch_size'], 'calib': batch['calib'], 'aug_param': batch['aug_param'],
          'virconv_proj': ops.projection_params(batch['calib'], batch['aug_param'], batch['batch_size'], DEV)}
    for s in STREAMS:
        vf0, vc0 = batch['voxel_features' + s], batch['voxel_coords' + s]
        n = vf0.shape[0]
        cap0 = (int(n * cap_margin) + grain - 1) // grain * grain
        vf = torch.full((cap0, vf0.shape[1]), tail, device=DEV)
        vc = torch.full((cap0, 4), -1.0, device=DEV)
        vf[:n], vc[:n] = vf0, vc0
        bd.update({'voxel_features' + s: vf, 'voxel_coords' + s: vc,
                   'virconv_static' + s: executor.StaticSpec(torch.tensor([n], dtype=torch.int32, device=DEV), caps[s],
                                                             torch.zeros(1, dtype=torch.int32, device=DEV))})
    return bd


@pytest.mark.parametrize('precision', ['bf16', 'fp32'])
def test_static_mode_matches_exact_mode(precision):
    """Same batch, same weights, BN in training mode: both streams in static mode publish the exact mode's nine tensors on
    the valid rows, zero / -1 tails beyond them, the same row counts, loss and parameter gradients."""
    from virconv_b200 import executor
    model = _model(precision)
    batch = _batch([11, 12])
    l0, g0, n0 = _exact(model, batch)
    caps = {s: executor.measured_caps(executor.last_run(model, s), 1.3, 256) for s in STREAMS}
    assert caps[''] and caps['_mm']
    for p in model.parameters():
        p.grad = None
    bd = _static_batch(batch, caps)
    out = model(bd)
    loss = _loss(out)
    loss.backward()
    torch.cuda.synchronize()
    for s in STREAMS:
        assert int(bd['virconv_static' + s].overflow.item()) == 0, s
    named = _named(out)
    assert len(named) == 9
    for k, t in named.items():
        e = n0[k]
        rows = int(t.num_rows.item())
        assert t.num_rows.dtype == torch.int32 and t.num_rows.is_cuda, k
        assert rows == e.features.shape[0], k
        assert t.features.shape[0] >= rows and t.features.shape[0] % 256 == 0, k
        assert torch.equal(t.indices[:rows].int(), e.indices.int()), k
        assert rel_err(t.features[:rows].detach().cpu(), e.features.detach().cpu()) < 1e-5, k
        if t.features.shape[0] > rows:
            assert float(t.features[rows:].abs().max()) == 0.0, k
            assert bool((t.indices[rows:] == -1).all()), k
    assert abs(float(loss) - l0) < 1e-5 * max(1.0, abs(l0))
    for name, p in model.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), name
        if precision == 'bf16':
            assert _grad_close(p.grad, g0[name]), name
        else:
            assert rel_err(p.grad.cpu(), g0[name].cpu()) < 2e-4, name


@pytest.mark.parametrize('stream', STREAMS)
def test_overflow_of_one_stream_is_reported_and_recaptured(stream, monkeypatch):
    """One strided conv's output set of one stream 300 rows short: that stream's flag reports the row count that did not
    fit, the other stream's stays 0; GraphedStep captured with such a capacity re-captures and then equals exact mode."""
    from virconv_b200 import executor
    from virconv_b200.graph import GraphedStep
    model = _model('bf16')
    batch = _batch([11, 12])
    l_e, g_e, _ = _exact(model, batch)
    caps = {s: executor.measured_caps(executor.last_run(model, s), 1.0, 1) for s in STREAMS}
    k = sorted(caps[stream])[0]
    true_rows = caps[stream][k]
    assert true_rows > 300
    caps[stream][k] = true_rows - 300
    bd = _static_batch(batch, caps, tail=0.0)
    with torch.no_grad():
        out = model(bd)
    torch.cuda.synchronize()
    for s in STREAMS:
        assert int(bd['virconv_static' + s].overflow.item()) == (true_rows if s == stream else 0), s
    for k_, t in _named(out).items():
        assert bool(torch.isfinite(t.features).all()), k_

    real = executor.measured_caps
    calls = []

    def tight(run, margin=1.3, grain=1024):          # the first capture's capacity of `stream` is 300 rows short
        c = real(run, margin, grain)
        calls.append(run)
        if len(calls) == STREAMS.index(stream) + 1:
            first = sorted(c)[0]
            c[first] = real(run, 1.0, 1)[first] - 300
        return c

    monkeypatch.setattr(executor, 'measured_caps', tight)
    step = GraphedStep(model, _loss, margin=1.3, grain=256)
    step(batch)
    torch.cuda.synchronize()
    assert step.recaptures == 1
    assert int(step.ovf_host[0, STREAMS.index(stream)]) == true_rows           # read back from the replay
    assert int(step.ovf_host[0, 1 - STREAMS.index(stream)]) == 0
    loss = step(batch)                                 # the flag of the previous replay -> re-capture, run this batch again
    torch.cuda.synchronize()
    assert step.recaptures == 2
    assert abs(float(loss) - l_e) < 1e-5 * max(1.0, abs(l_e))
    for name, p in model.named_parameters():
        assert _grad_close(p.grad, g_e[name]), name


def test_graph_replay_matches_exact_over_rotating_batches():
    """9 back-to-back replays over 4 batches, no host synchronisation between them: every step's loss and parameter gradients
    against an exact step of the same batch with the same weights."""
    from virconv_b200.graph import GraphedStep
    model = _model('bf16')
    batches = [_batch([20 + 2 * i, 21 + 2 * i]) for i in range(4)]
    ref = [_exact(model, b)[:2] for b in batches]
    step = GraphedStep(model, _loss, margin=1.35, grain=256)
    params = dict(model.named_parameters())
    got = []
    for s in range(9):
        loss = step(batches[s % 4])
        got.append((loss.detach().clone(), {k: v.grad.detach().clone() for k, v in params.items()}))
    torch.cuda.synchronize()
    assert step.recaptures == 1
    assert step.launches_per_replay > 0
    for s in range(9):
        l0, g0 = ref[s % 4]
        assert abs(float(got[s][0]) - l0) < 1e-5 * max(1.0, abs(l0)), s
        for k in params:
            assert _grad_close(got[s][1][k], g0[k]), (s, k)


def test_graph_with_in_graph_voxelisers():
    """Batches carry the collated `points` / `points_mm`; two vc_voxelize_mean calls (max-VFE for LiDAR, plain mean for the
    virtual points, per-stream voxel caps) run inside the graph.  Against the exact step on the host-voxelised batch of the
    same scenes."""
    from virconv_b200.graph import GraphedStep
    model = _model('bf16')
    ids = [[41, 42], [43, 44], [45, 46]]
    ref = [_exact(model, _batch(i))[:2] for i in ids]
    vox = dict(point_cloud_range=(0, -40, -3, 70.4, 40, 1), voxel_size=(0.05, 0.05, 0.05), max_points_per_voxel=5,
               max_voxels=MAX_VOXELS, vfe_model='max', max_voxels_mm=MAX_VOXELS, vfe_model_mm=None)
    step = GraphedStep(model, _loss, margin=1.35, grain=256, voxelizer=vox)
    params = dict(model.named_parameters())
    got = []
    for s in range(6):
        loss = step(_points_batch(ids[s % 3]))
        got.append((loss.detach().clone(), {k: v.grad.detach().clone() for k, v in params.items()}))
    torch.cuda.synchronize()
    assert step.recaptures == 1
    assert [st.cap0 for st in step.streams] == [2 * MAX_VOXELS, 2 * MAX_VOXELS]
    for s in range(6):
        l0, g0 = ref[s % 3]
        assert abs(float(got[s][0]) - l0) < 1e-5 * max(1.0, abs(l0)), s
        for k in params:
            assert _grad_close(got[s][1][k], g0[k]), (s, k)


def _valid(lists):
    out = []
    for t in lists:
        n = getattr(t, 'num_rows', None)
        out.append((t if n is None else t[:int(n)]).clone())
    return out


def test_captured_stvd_matches_module_path():
    """discard_mode='paper', discard_rng='device' in the captured step: the MM stream's four kept lists (sites 0-3) have the
    sizes int(n * (1 - rate)) over their input rows and ascending rows; the per-operator module path fed those lists
    publishes the same indices, features within 1e-4, fp32 parameter gradients within 2e-4."""
    from virconv_b200.graph import GraphedStep
    rate = CFG8['LAYER_DISCARD_RATE']
    model = _model('fp32', discard_mode='paper', discard_rng='device')
    twin = copy.deepcopy(model)
    batches = [_batch([50 + 2 * i, 51 + 2 * i]) for i in range(2)]
    holder = {}

    def loss_fn(out):
        holder['kept'], holder['named'] = out['stvd_kept_rows'], _named(out)
        return _loss(out)

    step = GraphedStep(model, loss_fn, margin=1.35, grain=256)
    params = dict(model.named_parameters())
    for s in range(4):
        batch = batches[s % 2]
        loss = step(batch)
        torch.cuda.synchronize()
        assert all(int(t.num_rows.item()) <= t.shape[0] for t in holder['kept'])
        kept = _valid(holder['kept'])
        named = {k: (t.features[:int(t.num_rows)].detach().clone(), t.indices[:int(t.num_rows)].clone())
                 for k, t in holder['named'].items()}
        l, g = float(loss), {k: v.grad.clone() for k, v in params.items()}
        for p in twin.parameters():
            p.grad = None
        bd = dict(batch)
        bd['stvd_keep_rows'] = kept
        out = twin(bd)
        ml = _loss(out)
        ml.backward()
        torch.cuda.synchronize()
        mn = _named(out)
        # list sizes: the float64 rule over each site's input rows (site 0: the input voxels; 1: vir_conv1 keeps the rows;
        # 2, 3: the strided conv of vir_conv2 / vir_conv3 over the previous site's kept rows)
        x1, x2 = mn['multi_scale_3d_features_mm:x_conv1'], mn['multi_scale_3d_features_mm:x_conv2']
        n_in = [batch['voxel_features_mm'].shape[0]]
        n_in.append(int(n_in[0] * (1.0 - rate)))
        n_in.append(orb.conv_rulebook(x1.indices.cpu().numpy(), x1.spatial_shape, 3, 2, 1)[0].shape[0])
        n_in.append(orb.conv_rulebook(x2.indices.cpu().numpy(), x2.spatial_shape, 3, 2, 1)[0].shape[0])
        assert len(kept) == 4
        for site, t in enumerate(kept):
            assert t.shape[0] == int(n_in[site] * (1.0 - rate)), (s, site)
            assert bool((t[1:] > t[:-1]).all()) and int(t[0]) >= 0 and int(t[-1]) < n_in[site], (s, site)
        for k, (f, idx) in named.items():
            assert torch.equal(idx.int(), mn[k].indices.int()), (s, k)
            assert rel_err(f.cpu(), mn[k].features.detach().cpu()) < 1e-4, (s, k)
        assert abs(l - float(ml)) < 1e-5 * max(1.0, abs(float(ml))), s
        for k, p in twin.named_parameters():
            assert rel_err(g[k].cpu(), p.grad.cpu()) < 2e-4, (s, k)
    assert step.recaptures == 1


def test_deterministic_replays_bit_identical():
    """torch.use_deterministic_algorithms(True), paper-mode StVD with a fixed stvd_seed: two replays of one batch from the
    same parameters and BatchNorm state agree bit for bit in the loss, every gradient and the BN running statistics."""
    from virconv_b200.graph import GraphedStep
    model = _model('bf16', discard_mode='paper', discard_rng='device')
    batch = _batch([5, 6])
    batch['stvd_seed'] = torch.tensor([1234], dtype=torch.int64, device=DEV)
    torch.use_deterministic_algorithms(True)
    try:
        step = GraphedStep(model, _loss, margin=1.3, grain=256)
        state = copy.deepcopy(model.state_dict())
        step(batch)                                    # capture (and one replay)
        torch.cuda.synchronize()
        recs = []
        for _ in range(2):
            model.load_state_dict(state)               # (in place: the graph keeps its parameter / buffer addresses)
            loss = step(batch)
            torch.cuda.synchronize()
            rec = {'loss': loss.detach().clone()}
            rec.update({'g:' + k: v.grad.clone() for k, v in model.named_parameters()})
            rec.update({'b:' + k: v.clone() for k, v in model.named_buffers()})
            recs.append(rec)
    finally:
        torch.use_deterministic_algorithms(False)
    assert step.recaptures == 1
    means = [k for k in state if k.endswith('running_mean')]
    assert means and all(not torch.equal(recs[0]['b:' + k], state[k]) for k in means)    # the replay updated them
    bad = [k for k in recs[0] if not torch.equal(recs[0][k], recs[1][k])]
    assert not bad, bad
