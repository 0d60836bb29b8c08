"""GPU tests of SyncBatchNorm on the fast path (sync_bn, vc_exec_forward_sync, vc_voxel_pool_bn_*_sync).

World size 1: a converted model computes bit for bit what the BatchNorm1d model computes, eagerly, in GraphedStep and in
GraphedForward.  Two ranks: two processes on this GPU with a gloo group; SyncBatchNorm over rank A = {scene a} and rank
B = {scene b} equals plain BatchNorm over the batch [a, b] (no convolution mixes scenes), which one process computes.
The captured step replays rank A's exchanges with rank B's recorded slots added in place of the all-reduce.

Run as a script, this file is the worker of one rank (argv: backend, init method, rank, world size, output path)."""
import copy
import os
import subprocess
import sys
from datetime import timedelta

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.testing import fill_module, rel_err  # noqa: E402

pytestmark = pytest.mark.gpu
CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG8 = dict(CFG, LAYER_DISCARD_RATE=0.15, MM=True)
SCENES = (20, 21)            # rank A, rank B; the union batch is [20, 21]
WORKER_TIMEOUT = 900


# ------------------------------------------------------------------------------------------------ shared by both sides
def _model(kind, precision, dev):
    from virconv_b200.backbone import VirConv8x, VirConvL8x
    m = (VirConvL8x(CFG, 8, [1408, 1600, 80], precision=precision) if kind == 'L'
         else VirConv8x(CFG8, 8, [1408, 1600, 80], precision=precision))
    fill_module(m, 666 if kind == 'L' else 667)
    return m.to(dev).train()


def _sync(m):
    return torch.nn.SyncBatchNorm.convert_sync_batchnorm(m)


def _batch(kind, ids, dev, training=True, size=(4096, 9000, 7000)):
    from virconv_b200 import scenes
    if kind == 'L':
        b = scenes.make_batch(ids, n_lidar=size[0], n_virtual=size[1], max_voxels=size[2], training=training)
        bd = {'voxel_features': torch.from_numpy(b.voxel_features.copy()).to(dev),
              'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).to(dev), 'batch_size': b.batch_size, 'calib': b.calib}
        if training:
            bd['aug_param'] = torch.from_numpy(b.aug_param.copy())
        return bd
    b = scenes.make_batch_mm(ids, max_voxels=3000, training=True, n_lidar=4096, n_virtual=6000)
    bd = {k: torch.from_numpy(v.copy()).to(dev) for k, v in b.arrays.items()}
    bd.update(batch_size=b.batch_size, calib=b.calib, aug_param=torch.from_numpy(b.aug_param.copy()))
    return bd


def _named(out):
    named = {}
    for g in ('multi_scale_3d_features', 'multi_scale_3d_features_mm'):
        named.update({f'{g}:{k}': t for k, t in out.get(g, {}).items()})
    named['out'] = out['encoded_spconv_tensor']
    return named


def _weight(t):
    """A fixed per-row, per-channel weight from the voxel's (z, y, x) — not its batch index, so that scene b weighs the same
    as batch 0 of rank B and as batch 1 of the union.  Capacity tails (index -1) weigh nothing (their features are 0).
    Positive (1 +- 0.5): with weights of both signs the parameter gradients would be sums that cancel to ~sqrt(rows), and
    one activation that a last-bit difference moves across the ReLU would show as a relative error of ~1/sqrt(rows)."""
    zyx = t.indices[:, 1:].double()
    c = torch.arange(t.features.shape[1], device=zyx.device, dtype=torch.float64)
    return (1.0 + 0.5 * torch.cos(0.37 * zyx[:, 2:3] + 0.11 * zyx[:, 1:2] + 0.05 * zyx[:, 0:1] + 0.7 * c)).float()


def _loss(out):
    """A sum over rows: the union's loss is the sum of the ranks' losses, and so are the parameter gradients."""
    return sum((t.features * _weight(t)).sum() for t in _named(out).values())


def _record(model, out_loss, out):
    return {'loss': float(out_loss.detach()),
            'feats': {k: (t.features.detach().cpu(), t.indices.detach().cpu()) for k, t in _named(out).items()},
            'grads': {k: p.grad.detach().cpu().clone() for k, p in model.named_parameters()},
            'bufs': {k: b.detach().cpu().clone() for k, b in model.named_buffers()}}


def _eager(model, batch):
    for p in model.parameters():
        p.grad = None
    out = model(dict(batch))
    loss = _loss(out)
    loss.backward()
    torch.cuda.synchronize()
    return _record(model, loss, out)


def _pool_inputs(dev):
    from oracle import voxel_pool_golden as g
    from test_cpu_voxel_pool import golden, golden_inputs
    x = {k: (v.float() if v.is_floating_point() else v).to(dev) for k, v in golden_inputs(golden()).items()}
    nc = x['new_coords']
    C = g.CFG['mlps'][0][1]
    gen = torch.Generator().manual_seed(5)
    return dict(xyz=x['xyz'].contiguous(), new_xyz=x['new_xyz'].contiguous(),
                new_coords=torch.cat([nc[:, :1], nc[:, 1:].flip(1)], 1).int().contiguous(), v2p=x['voxel2point_indices'].int(),
                feats=torch.randn(x['xyz'].shape[0], C, generator=gen).to(dev),
                w_out=torch.randn(nc.shape[0], C, generator=gen).to(dev), C=C, max_range=g.CFG['query_ranges'][0],
                radius=g.CFG['radii'][0], nsample=g.CFG['nsamples'][0])


def _pool(rows, sync, dev):
    """One voxel_pool call over the query points `rows` with a fresh position branch (SyncBatchNorm2d when sync)."""
    from virconv_b200.voxel_pool import voxel_pool
    x = _pool_inputs(dev)
    torch.manual_seed(7)
    mlp = torch.nn.Sequential(torch.nn.Conv2d(3, x['C'], 1, bias=False), torch.nn.BatchNorm2d(x['C']))
    torch.nn.init.normal_(mlp[1].weight, 1.0, 0.2)
    torch.nn.init.normal_(mlp[1].bias, 0.0, 0.2)
    mlp = (_sync(mlp) if sync else mlp).to(dev).train()
    f = x['feats'].clone().requires_grad_(True)
    pooled = voxel_pool(f, x['xyz'], x['new_xyz'][rows], x['new_coords'][rows], x['v2p'], mlp, x['max_range'], x['radius'],
                        x['nsample'])[0]
    (pooled * x['w_out'][rows]).sum().backward()
    torch.cuda.synchronize()
    return {'pooled': pooled.detach().cpu(), 'dfeat': f.grad.cpu(), 'dw': mlp[0].weight.grad.cpu(),
            'dgamma': mlp[1].weight.grad.cpu(), 'dbeta': mlp[1].bias.grad.cpu(), 'rm': mlp[1].running_mean.cpu(),
            'rv': mlp[1].running_var.cpu()}


def _pool_rows(rank, world, dev):
    m = _pool_inputs(dev)['new_xyz'].shape[0]
    return torch.arange(m, device=dev)[rank::world] if world > 1 else torch.arange(m, device=dev)


# ------------------------------------------------------------------------------------------------ worker (one rank)
def _worker(backend, init, rank, world, out_path):
    import torch.distributed as dist
    dev = torch.device('cuda:%d' % (0 if backend == 'gloo' else rank))
    torch.cuda.set_device(dev)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    dist.init_process_group(backend, init_method=init, rank=rank, world_size=world, timeout=timedelta(seconds=600))
    res = {}
    try:
        if backend == 'gloo':
            for name, kind, prec in (('L', 'L', 'fp32'), ('T', 'T', 'fp32'), ('Lbf16', 'L', 'bf16')):
                model = _sync(_model(kind, prec, dev))
                rec = {}

                def reducer(slot, key, rec=rec):         # rank B's slots before the sum, for the captured test
                    rec[key] = slot.detach().cpu().clone()
                    dist.all_reduce(slot)
                model.bn_reducer = reducer
                res[name] = _eager(model, _batch(kind, [SCENES[rank]], dev))
                res[name]['slots'] = rec
            prev = torch.are_deterministic_algorithms_enabled()
            torch.use_deterministic_algorithms(True)
            try:
                res['det'] = [_eager(_sync(_model('L', 'bf16', dev)), _batch('L', [SCENES[rank]], dev)) for _ in range(2)]
            finally:
                torch.use_deterministic_algorithms(prev)
            res['pool'] = _pool(_pool_rows(rank, world, dev), True, dev)
            res['regrow'] = _regrow(rank, dev)
        else:                                            # NCCL, one GPU per rank: the captured step
            from virconv_b200.graph import GraphedStep
            model = _sync(_model('L', 'fp32', dev))
            keep = {}

            def loss_fn(out):
                keep['out'] = out
                return _loss(out)
            step = GraphedStep(model, loss_fn, margin=1.35, grain=256)
            batch = _batch('L', [SCENES[rank]], dev)
            bufs0 = {k: b.detach().clone() for k, b in model.named_buffers()}
            step(batch)                                   # exact run, warm-up, capture
            for k, b in model.named_buffers():
                b.copy_(bufs0[k])
            loss = step(batch)                           # one replay from the initial running statistics
            torch.cuda.synchronize()
            res['graph'] = _record(model, loss, keep['out'])
    finally:
        dist.destroy_process_group()
    torch.save(res, out_path)


def _regrow(rank, dev):
    """GraphedStep over two calls: rank A's second batch does not fit the input buffers (it must grow and re-capture), rank
    B's is its first batch again.  The reducer only counts the exchanges (a gloo all-reduce cannot be captured); a rank that
    re-captured alone would issue more of them than the other."""
    from virconv_b200.graph import GraphedStep
    model = _sync(_model('L', 'bf16', dev))
    calls = [0]

    def count(slot, key):
        calls[0] += 1
    model.bn_reducer = count
    step = GraphedStep(model, _loss, margin=1.05, grain=64)
    small = _batch('L', [31 + rank], dev, size=(2048, 3000, 2500))
    big = _batch('L', [33], dev, size=(4096, 9000, 7000)) if rank == 0 else small
    losses = [float(step(small)), float(step(big))]
    torch.cuda.synchronize()
    return {'recaptures': step.recaptures, 'exchanges': calls[0], 'losses': losses}


# ------------------------------------------------------------------------------------------------ the test process
def _launch(tmp_path, backend='gloo'):
    """Run the two ranks as child processes and collect their results; nothing outlives the call."""
    init = 'file://' + str(tmp_path / 'rendezvous')
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    flags = ['-s'] if sys.flags.no_user_site else []
    procs = [subprocess.Popen([sys.executable, *flags, os.path.abspath(__file__), backend, init, str(r), '2',
                               str(tmp_path / ('rank%d.pt' % r))], env=env, cwd=ROOT, stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT) for r in range(2)]
    logs = []
    try:
        for p in procs:
            logs.append(p.communicate(timeout=WORKER_TIMEOUT)[0].decode(errors='replace'))
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    for p, log in zip(procs, logs):
        assert p.returncode == 0, log[-4000:]
    return [torch.load(tmp_path / ('rank%d.pt' % r), weights_only=False) for r in range(2)]


@pytest.fixture(scope='module')
def two_ranks(lib_built, tmp_path_factory):
    return _launch(tmp_path_factory.mktemp('sync_bn'))


@pytest.fixture(scope='module')
def union(lib_built):
    """Plain BatchNorm over the union batch, one process."""
    dev = torch.device('cuda:0')
    res = {name: _eager(_model(kind, prec, dev), _batch(kind, list(SCENES), dev))
           for name, kind, prec in (('L', 'L', 'fp32'), ('T', 'T', 'fp32'), ('Lbf16', 'L', 'bf16'))}
    # bf16: the union batch with its scenes swapped — the same sums over a different partition of the rows, which is what
    # splitting them over ranks changes; the comparison is held to that noise (the loss does not see the batch order)
    res['Lbf16_swapped'] = _eager(_model('L', 'bf16', dev), _batch('L', list(SCENES[::-1]), dev))
    res['pool'] = _pool(_pool_rows(0, 1, dev), False, dev)
    return res


def _rows_of(feats, idx, b):
    """The rows of batch index b, sorted by (z, y, x) -> (features, zyx)."""
    keep = idx[:, 0] == b
    f, zyx = feats[keep], idx[keep][:, 1:].long()
    key = (zyx[:, 0] * 4096 + zyx[:, 1]) * 4096 + zyx[:, 2]
    order = torch.argsort(key)
    return f[order], zyx[order]


def _errs(got, ref):
    got, ref = got.double(), ref.double()
    return float((got - ref).norm() / ref.norm().clamp_min(1e-30)), rel_err(got, ref)


def _grad_close(got, ref, swapped):
    """bf16: the criterion of tests/test_gpu_graph.py (relative L2 below 1e-2, largest difference below 3e-2 of the largest
    element), or, where it is larger, within 4x the difference between the union batch and the same batch with its scenes
    swapped (`swapped`): bf16 rounding of activations and gradients amplifies every last-bit change of a reordered sum
    from layer to layer."""
    l2, mx = _errs(got, ref)
    n_l2, n_mx = _errs(swapped, ref)
    return l2 < max(1e-2, 4 * n_l2) and mx < max(3e-2, 4 * n_mx), (l2, mx, n_l2, n_mx)


@pytest.mark.parametrize('name', ['L', 'T', 'Lbf16'])
def test_two_ranks_match_the_union_batch(two_ranks, union, name):
    bf16 = name.endswith('bf16')
    ref = union[name]
    ranks = [r[name] for r in two_ranks]
    for b, rk in enumerate(ranks):
        for k, (f, idx) in rk['feats'].items():
            fr, zr = _rows_of(*ref['feats'][k], b)
            fg, zg = _rows_of(f, idx, 0)
            assert torch.equal(zg, zr), (k, b)
            assert rel_err(fg, fr) <= (3e-2 if bf16 else 1e-4), (k, b, rel_err(fg, fr))
    for k, v in ranks[0]['bufs'].items():
        assert torch.equal(v, ranks[1]['bufs'][k]), k
        if v.is_floating_point():
            assert float((v.double() - ref['bufs'][k].double()).abs().max()) <= (1e-3 if bf16 else 1e-5), k
        else:
            assert int(v) == int(ref['bufs'][k]), k
    for k, g0 in ref['grads'].items():
        got = ranks[0]['grads'][k] + ranks[1]['grads'][k]
        if bf16:
            ok, errs = _grad_close(got, g0, union['Lbf16_swapped']['grads'][k])
            assert ok, (k, errs)
        else:
            assert rel_err(got, g0) <= 2e-3, (k, rel_err(got, g0))


def test_two_ranks_deterministic_runs_are_bit_identical(two_ranks):
    for r in two_ranks:
        a, b = r['det']
        assert a['loss'] == b['loss']
        for part in ('grads', 'bufs'):
            for k in a[part]:
                assert torch.equal(a[part][k], b[part][k]), (part, k)
        for k in a['feats']:
            assert torch.equal(a['feats'][k][0], b['feats'][k][0]) and torch.equal(a['feats'][k][1], b['feats'][k][1]), k


def test_two_ranks_voxel_pool_matches_the_union(two_ranks, union):
    ref = union['pool']
    m = ref['pooled'].shape[0]
    for r, res in enumerate(two_ranks):
        assert rel_err(res['pool']['pooled'], ref['pooled'][torch.arange(m)[r::2]]) <= 1e-5
        assert torch.equal(res['pool']['rm'], two_ranks[0]['pool']['rm'])
        assert float((res['pool']['rm'] - ref['rm']).abs().max()) <= 1e-5
        assert float((res['pool']['rv'] - ref['rv']).abs().max()) <= 1e-5
    for k in ('dw', 'dgamma', 'dbeta', 'dfeat'):
        got = two_ranks[0]['pool'][k] + two_ranks[1]['pool'][k]
        assert rel_err(got, ref[k]) <= 1e-5, (k, rel_err(got, ref[k]))


def test_ranks_grow_and_recapture_together(two_ranks):
    """One rank's batch outgrows its capture: every rank re-captures, and all issue the same number of exchanges."""
    a, b = two_ranks[0]['regrow'], two_ranks[1]['regrow']
    assert a['recaptures'] == b['recaptures'] == 2
    assert a['exchanges'] == b['exchanges']
    assert all(abs(v) < float('inf') for v in a['losses'] + b['losses'])


def test_captured_step_replays_the_exchange(two_ranks):
    """Rank A's GraphedStep with a reducer that adds rank B's recorded slots matches rank A's eager two-rank step."""
    from virconv_b200.graph import GraphedStep
    dev = torch.device('cuda:0')
    want = two_ranks[0]['L']
    slots = {k: v.to(dev) for k, v in two_ranks[1]['L']['slots'].items()}
    model = _sync(_model('L', 'fp32', dev))
    model.bn_reducer = lambda slot, key: slot.add_(slots[key])
    keep = {}

    def loss_fn(out):
        keep['out'] = out
        return _loss(out)
    step = GraphedStep(model, loss_fn, margin=1.35, grain=256)
    batch = _batch('L', [SCENES[0]], dev)
    bufs0 = {k: b.detach().clone() for k, b in model.named_buffers()}
    step(batch)
    for k, b in model.named_buffers():
        b.copy_(bufs0[k])
    loss = step(batch)
    torch.cuda.synchronize()
    got = _record(model, loss, keep['out'])
    assert abs(got['loss'] - want['loss']) <= 1e-5 * max(1.0, abs(want['loss']))
    for k, (f, idx) in got['feats'].items():
        fg, zg = _rows_of(f, idx, 0)
        fw, zw = _rows_of(*want['feats'][k], 0)
        assert torch.equal(zg, zw), k
        assert rel_err(fg, fw) <= 1e-4, k
    for k, v in want['bufs'].items():
        if v.is_floating_point():
            assert float((got['bufs'][k].double() - v.double()).abs().max()) <= 1e-5, k
        else:
            assert int(got['bufs'][k]) == int(v), k
    for k, g in want['grads'].items():
        assert rel_err(got['grads'][k], g) <= 2e-3, (k, rel_err(got['grads'][k], g))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two GPUs')
def test_nccl_graphed_step_world_size_two(lib_built, union, tmp_path):
    """Two GPUs, NCCL: each rank's captured step (the all-reduce captured in the graph) against the union oracle."""
    ranks = [r['graph'] for r in _launch(tmp_path, 'nccl')]
    ref = union['L']
    for b, rk in enumerate(ranks):
        for k, (f, idx) in rk['feats'].items():
            fr, zr = _rows_of(*ref['feats'][k], b)
            fg, zg = _rows_of(f, idx, 0)
            assert torch.equal(zg, zr) and rel_err(fg, fr) <= 1e-4, k
    for k, g0 in ref['grads'].items():
        assert rel_err(ranks[0]['grads'][k] + ranks[1]['grads'][k], g0) <= 2e-3, k


# ------------------------------------------------------------------------------------------------ world size 1
@pytest.fixture
def det_mode():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


def _assert_same(a, b):
    assert a['loss'] == b['loss']
    for part in ('grads', 'bufs'):
        for k in a[part]:
            assert torch.equal(a[part][k], b[part][k]), (part, k)
    for k in a['feats']:
        assert torch.equal(a['feats'][k][0], b['feats'][k][0]) and torch.equal(a['feats'][k][1], b['feats'][k][1]), k


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_world_size_one_is_batchnorm_bit_for_bit(lib_built, det_mode, precision):
    """Without a process group SyncBatchNorm is BatchNorm: the converted model runs the plan (the deterministic flag does
    not raise) with the same kernels — eager, in GraphedStep and in GraphedForward."""
    from virconv_b200.graph import GraphedForward, GraphedStep
    dev = torch.device('cuda:0')
    plain = _model('L', precision, dev)
    conv = _sync(copy.deepcopy(plain))
    assert conv._use_plan(_batch('L', [SCENES[0]], dev)['voxel_features'])
    batch = _batch('L', list(SCENES), dev)
    _assert_same(_eager(conv, batch), _eager(plain, batch))

    rec = []
    for m in (plain, conv):
        keep = {}

        def loss_fn(out, keep=keep):
            keep['out'] = out
            return _loss(out)
        step = GraphedStep(m, loss_fn, margin=1.35, grain=256)
        step(batch)
        loss = step(batch)
        torch.cuda.synchronize()
        rec.append(_record(m, loss, keep['out']))
    _assert_same(rec[0], rec[1])

    outs = []
    for m in (plain, conv):
        m.eval()
        out = GraphedForward(m, margin=1.35, grain=256)(_batch('L', list(SCENES), dev, training=False))
        torch.cuda.synchronize()
        outs.append({k: (t.features.cpu().clone(), t.indices.cpu().clone()) for k, t in _named(out).items()})
    for k in outs[0]:
        assert torch.equal(outs[0][k][0], outs[1][k][0]) and torch.equal(outs[0][k][1], outs[1][k][1]), k


if __name__ == '__main__':
    _worker(sys.argv[1], sys.argv[2], int(sys.argv[3]), int(sys.argv[4]), sys.argv[5])
