"""GPU tests of the fused parameter update (vc_optim_step, optim.FusedAdamOneCycle) and of the captured step that ends
with it: against the float64 restatement, the reference's recorded run (tests/golden/optim_ref.npz) and the same update
done with torch (clip_grad_norm_, one mul_ per tensor, torch.optim.Adam)."""
import os

import numpy as np
import pytest
import torch

from oracle import optim as ooptim
from oracle import optim_golden as og
from oracle.testing import fill_module

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device('cuda:0')
CFG_L = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG_T = dict(CFG_L, LAYER_DISCARD_RATE=0.15, MM=True)


@pytest.fixture(autouse=True)
def _built(lib_built):
    yield
    from virconv_b200 import ops
    torch.cuda.synchronize()
    assert int(ops.tc_error_flag(DEV).item()) == 0


def _rel(got, want):
    got = got.detach().double().cpu().numpy() if torch.is_tensor(got) else np.asarray(got, dtype=np.float64)
    want = want.detach().double().cpu().numpy() if torch.is_tensor(want) else np.asarray(want, dtype=np.float64)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def _torch_step(groups, adam, lr, mom, wd, max_norm, clip_params):
    """The reference's update over torch: clip, true weight decay one tensor at a time, Adam with this step's momentum."""
    norm = None
    if max_norm is not None:
        norm = torch.nn.utils.clip_grad_norm_(clip_params, max_norm)
    with torch.no_grad():
        for g in groups:
            for p in g:
                p.mul_(1 - wd * lr)
    for g in adam.param_groups:
        g['lr'], g['betas'], g['weight_decay'] = lr, (mom, 0.99), 0
    adam.step()
    return norm


def _torch_arm(model):
    from virconv_b200.optim import leaf_param_groups
    groups, _ = leaf_param_groups(model)
    return groups, torch.optim.Adam([{'params': g, 'lr': 0} for g in groups], betas=(0.9, 0.99))


def test_golden_tree_step_by_step():
    """The reference's own 40 iterations: total norm within 1e-6 of the float64 restatement at every step; parameters, m and v
    no further from it than twice what the torch arm on the same GPU is (and never beyond 1e-5), and on the recorded run."""
    from virconv_b200.optim import FusedAdamOneCycle
    gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'optim_ref.npz'))
    wd = og.CFG['WEIGHT_DECAY']
    model, twin = og.golden_tree().to(DEV), og.golden_tree().to(DEV)
    named, tnamed = dict(model.named_parameters()), dict(twin.named_parameters())
    opt = FusedAdamOneCycle.from_model(model, wd=wd)
    names = [str(n) for n in list(gold['group0']) + list(gold['group1'])]
    assert [id(p) for p in opt.params] == [id(named[n]) for n in names] and opt.norm_only[0] is named['block.scale']
    tgroups, adam = _torch_arm(twin)
    o = ooptim.AdamOneCycle([gold['init.' + n] for n in names], wd=wd)
    worst = {'fused': 0.0, 'torch': 0.0}
    for it in range(og.STEPS):
        lr, mom = float(gold['lr'][it]), float(gold['mom'][it])
        g = og.golden_grads(model, it)
        for n, v in g.items():
            named[n].grad = torch.from_numpy(v.copy()).to(DEV)
            tnamed[n].grad = torch.from_numpy(v.copy()).to(DEV)
        kept = {n: named[n].grad.clone() for n in g}
        opt.lr, opt.mom = lr, mom
        opt.step(max_norm=og.MAX_NORM)
        tnorm = _torch_step(tgroups, adam, lr, mom, wd, og.MAX_NORM, list(twin.parameters()))
        o.step([g.get(n) for n in names], lr, mom, og.MAX_NORM, norm_only=[v for n, v in g.items() if n not in names])
        assert abs(float(opt.last_total_norm) - o.total_norm) <= 1e-6 * o.total_norm, it
        assert abs(float(opt.last_total_norm) - float(gold['total_norm'][it])) <= 1e-6 * o.total_norm, it
        assert abs(float(tnorm) - o.total_norm) <= 1e-5 * o.total_norm
        assert all(torch.equal(named[n].grad, kept[n]) for n in g), 'step() modified a gradient'
        for i, n in enumerate(names):
            worst['fused'] = max(worst['fused'], _rel(named[n], o.p[i]), _rel(opt.state[named[n]]['exp_avg'], o.m[i]),
                                 _rel(opt.state[named[n]]['exp_avg_sq'], o.v[i]))
            st = adam.state.get(tnamed[n])
            worst['torch'] = max(worst['torch'], _rel(tnamed[n], o.p[i]),
                                 *([_rel(st['exp_avg'], o.m[i]), _rel(st['exp_avg_sq'], o.v[i])] if st else []))
        if it + 1 in og.CHECKPOINTS:
            for n in names:
                assert _rel(named[n], gold['p.%d.%s' % (it + 1, n)]) < 2e-6, (it, n)
    assert worst['fused'] <= max(2 * worst['torch'], 2e-7) and worst['fused'] < 1e-5, worst
    assert opt.applied_steps() == og.STEPS and opt.skipped_steps() == 0
    assert torch.equal(named['block.scale'].cpu(), torch.from_numpy(gold['init.block.scale']))       # counted, never updated
    assert torch.equal(named['frozen.weight'].cpu(), torch.from_numpy(gold['init.frozen.weight']))
    # the decay-only tensors: (1 - wd * lr) every step, no Adam state
    assert not opt.state[named['unused.weight']]['exp_avg'].any()
    sd = opt.state_dict()
    assert sorted(sd['state']) == gold['sd_state_keys'].tolist() and sd['param_groups'][1]['params'] == gold['sd_group1'].tolist()


def _detector_sized():
    """The tensors of a real VirConv8x plus synthetic ones up to ~13 M elements: an 8 M and a 3 M + 1 tensor, views that
    start 4 and 8 bytes past a 16-byte boundary, a 1-element tensor."""
    from virconv_b200.backbone import VirConv8x
    m = VirConv8x(CFG_T, 8, [1408, 1600, 80])
    fill_module(m, 668)
    params = [p for p in m.to(DEV).parameters()]
    gen = torch.Generator(device='cpu').manual_seed(5)
    for n, shift in ((8 << 20, 0), ((3 << 20) + 1, 0), (70001, 1), (4099, 2), (1, 0), (5, 3)):
        buf = (torch.randn(n + shift, generator=gen) * 0.05).to(DEV)
        params.append(torch.nn.Parameter(buf[shift:]))
    assert params[-4].data_ptr() % 16 == 4 and params[-3].data_ptr() % 16 == 8
    return params


def _rand_grads(params, seed, scale=1e-3, skip=()):
    gen = torch.Generator(device='cpu').manual_seed(seed)
    return [None if i in skip else (torch.randn(p.numel(), generator=gen) * scale).view_as(p).to(DEV) for i, p in enumerate(params)]


def test_detector_sized_set_bit_equality_and_launches():
    from virconv_b200 import _lib
    from virconv_b200.optim import FusedAdamOneCycle
    params = _detector_sized()
    assert sum(p.numel() for p in params) > 12_000_000
    p0 = [p.detach().clone() for p in params]
    skip = (3, len(params) - 1)                                    # two tensors never receive a gradient: decayed only
    o = ooptim.AdamOneCycle([p.cpu().numpy() for p in p0], wd=0.01)
    runs = []
    for max_ctas in (0, 0, 37):                                    # twice the same, then another grid: all bit-identical
        with torch.no_grad():
            for p, q in zip(params, p0):
                p.copy_(q)
        opt = FusedAdamOneCycle(params, wd=0.01, max_ctas=max_ctas)
        norms = []
        for it in range(3):
            grads = _rand_grads(params, 100 + it, 1e-3 if it != 1 else 1.0, skip)
            for p, g in zip(params, grads):
                p.grad = g
            opt.lr, opt.mom = 0.003 * (it + 1), 0.95 - 0.01 * it
            l0 = _lib.load().vc_launch_count()
            opt.step(max_norm=None if it == 2 else 10.0)
            assert _lib.load().vc_launch_count() - l0 <= 2
            norms.append(opt.last_total_norm.clone())
            if not runs:
                o.step([None if g is None else g.cpu().numpy() for g in grads], opt.lr, opt.mom, None if it == 2 else 10.0)
                assert abs(float(norms[-1]) - o.total_norm) <= 1e-6 * o.total_norm
                assert (o.clip_coef < 1.0) == (it == 1)
        torch.cuda.synchronize()
        runs.append(([p.detach().clone() for p in params], opt.exp_avg_flat.clone(), opt.exp_avg_sq_flat.clone(), norms))
        if len(runs) == 1:
            for i, p in enumerate(params):
                assert _rel(p, o.p[i]) < 1e-5, i
                assert _rel(opt.state[p]['exp_avg'], o.m[i]) < 1e-5 and _rel(opt.state[p]['exp_avg_sq'], o.v[i]) < 1e-5, i
            for i in skip:
                assert not opt.state[params[i]]['exp_avg'].any()
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(r[0], runs[0][0]))
        assert torch.equal(r[1], runs[0][1]) and torch.equal(r[2], runs[0][2])
        assert all(torch.equal(a, b) for a, b in zip(r[3], runs[0][3]))


def test_guard_skips_and_the_next_step_applies():
    from virconv_b200.optim import FusedAdamOneCycle
    params = [torch.nn.Parameter(torch.randn(5000, device=DEV)), torch.nn.Parameter(torch.randn(7, 3, device=DEV))]
    word = torch.zeros(2, dtype=torch.int32, device=DEV)            # a private guard, not the library's error flag
    opt = FusedAdamOneCycle(params, lr=0.01, wd=0.01, guards=[word])
    twin = [torch.nn.Parameter(p.detach().clone()) for p in params]
    ref = FusedAdamOneCycle(twin, lr=0.01, wd=0.01)

    def step_both(seed, poison=None, raise_word=False):
        grads = _rand_grads(params, seed)
        for p, q, g in zip(params, twin, grads):
            p.grad, q.grad = g.clone(), g.clone()
        if poison is not None:
            params[0].grad[123] = poison
        word[1] = 7 if raise_word else 0
        opt.step(max_norm=10.0)
        if poison is None and not raise_word:
            ref.step(max_norm=10.0)

    step_both(1)
    for kw in (dict(poison=float('inf')), dict(poison=float('nan')), dict(raise_word=True)):
        before = [p.detach().clone() for p in params] + [opt.exp_avg_flat.clone(), opt.exp_avg_sq_flat.clone()]
        n_skip = opt.skipped_steps()
        step_both(2, **kw)
        after = [p.detach() for p in params] + [opt.exp_avg_flat, opt.exp_avg_sq_flat]
        assert all(torch.equal(a, b) for a, b in zip(before, after)), kw
        assert opt.skipped_steps() == n_skip + 1 and opt.applied_steps() == 1
        if 'poison' in kw:
            assert not np.isfinite(float(opt.last_total_norm))
    step_both(3)                                                    # applies with t = 2, as if the skipped steps never were
    assert opt.applied_steps() == 2 == ref.applied_steps() and opt.skipped_steps() == 3
    assert all(torch.equal(p, q) for p, q in zip(params, twin)) and torch.equal(opt.exp_avg_flat, ref.exp_avg_flat)


def test_step_makes_no_host_read_and_follows_moving_gradients():
    """step() under torch's sync debug mode, with new gradient tensors (new addresses) and new lr / mom every step, and with
    a tensor that loses its gradient half way; the result equals a run whose gradients stay where they are."""
    from virconv_b200.optim import FusedAdamOneCycle
    shapes = [(64, 27, 32), (33,), (1,), (4097,)]
    gen = torch.Generator(device='cpu').manual_seed(9)
    init = [torch.randn(s, generator=gen) for s in shapes]
    a = [torch.nn.Parameter(t.clone().to(DEV)) for t in init]
    b = [torch.nn.Parameter(t.clone().to(DEV)) for t in init]
    oa, ob = FusedAdamOneCycle(a, wd=0.01), FusedAdamOneCycle(b, wd=0.01)
    fixed = [torch.zeros_like(p) for p in b]
    for p, g in zip(b, fixed):
        p.grad = g
    hold = []
    for it in range(12):
        grads = _rand_grads(a, 50 + it, 0.1)
        hold.append(grads)                                          # (kept alive: every step sees fresh addresses)
        for p, g, f in zip(a, grads, fixed):
            p.grad = g
            f.copy_(g)
        if it >= 6:
            a[1].grad, b[1].grad = None, None
        for o in (oa, ob):
            o.lr, o.mom = 0.001 * (it + 1), 0.95 - 0.005 * it
        torch.cuda.set_sync_debug_mode('error')
        try:
            oa.step(max_norm=1.0)
        finally:
            torch.cuda.set_sync_debug_mode('default')
        ob.step(max_norm=1.0)
    assert oa.applied_steps() == 12
    assert all(torch.equal(p, q) for p, q in zip(a, b)) and torch.equal(oa.exp_avg_sq_flat, ob.exp_avg_sq_flat)


def test_refusals():
    from virconv_b200.optim import FusedAdamOneCycle
    with pytest.raises(ValueError, match='fp32'):
        FusedAdamOneCycle([torch.nn.Parameter(torch.zeros(4, device=DEV, dtype=torch.float64))])
    frozen = torch.nn.Parameter(torch.zeros(4, device=DEV), requires_grad=False)
    with pytest.raises(ValueError, match='no trainable'):
        FusedAdamOneCycle([frozen])
    p = torch.nn.Parameter(torch.zeros(4, 4, device=DEV))
    opt = FusedAdamOneCycle([p, frozen])
    assert len(opt.params) == 1 and opt.params[0] is p
    p.grad = torch.zeros(4, 8, device=DEV)[:, ::2]                  # not contiguous
    with pytest.raises(ValueError, match='gradient'):
        opt.step()
    with pytest.raises(ValueError, match='guard words'):
        opt.bind([torch.zeros(9, dtype=torch.int32, device=DEV)])


def test_checkpoint_round_trip_with_torch_adam():
    """Five fused steps -> state_dict -> torch.optim.Adam.load_state_dict -> one torch step equals one more fused step;
    Adam's state_dict -> a fresh fused optimizer -> the step after that agrees too."""
    from virconv_b200.optim import FusedAdamOneCycle
    wd = 0.01
    model, twin = og.golden_tree().to(DEV), og.golden_tree().to(DEV)
    named, tnamed = dict(model.named_parameters()), dict(twin.named_parameters())
    opt = FusedAdamOneCycle.from_model(model, wd=wd)

    def load_grads(it, *nameds):
        for n, v in og.golden_grads(model, it).items():
            for nd in nameds:
                nd[n].grad = torch.from_numpy(v.copy()).to(DEV)

    for it in range(5):
        load_grads(it, named)
        opt.lr, opt.mom = 0.002, 0.93
        opt.step(max_norm=og.MAX_NORM)
    twin.load_state_dict(model.state_dict())
    tgroups, adam = _torch_arm(twin)
    adam.load_state_dict(opt.state_dict())
    load_grads(5, named, tnamed)
    opt.step(max_norm=og.MAX_NORM)
    _torch_step(tgroups, adam, 0.002, 0.93, wd, og.MAX_NORM, list(twin.parameters()))
    assert all(_rel(tnamed[n], p) < 1e-6 for n, p in named.items())
    fresh_model = og.golden_tree().to(DEV)
    fresh_model.load_state_dict(twin.state_dict())
    fresh = FusedAdamOneCycle.from_model(fresh_model, wd=wd)
    fresh.load_state_dict(adam.state_dict())
    assert fresh.applied_steps() == 6 and fresh.lr == 0.002 and fresh.mom == 0.93
    fnamed = dict(fresh_model.named_parameters())
    load_grads(6, named, fnamed)
    opt.step(max_norm=og.MAX_NORM)
    fresh.step(max_norm=og.MAX_NORM)
    assert all(_rel(fnamed[n], p) < 1e-6 for n, p in named.items())
    assert _rel(fresh.exp_avg_flat, opt.exp_avg_flat) < 1e-6


def test_reference_clip_name_records_for_the_owning_optimizer():
    import virconv_b200.reference_env as renv
    from virconv_b200.optim import FusedAdamOneCycle
    a = [torch.nn.Parameter(torch.ones(64, device=DEV))]
    b = [torch.nn.Parameter(torch.ones(64, device=DEV))]
    oa, ob = FusedAdamOneCycle(a, wd=0.0), FusedAdamOneCycle(b, wd=0.0)
    for p in a + b:
        p.grad = torch.full((64,), 2.0, device=DEV)
    assert renv._fused_clip_grad_norm_(a, 4.0) is None and torch.equal(a[0].grad, b[0].grad)      # gradients left alone
    oa.step()
    ob.step()
    assert abs(float(oa._status[1]) - 0.25) < 1e-6 and float(ob._status[1]) == 1.0                  # clip_coef: 4 / 16, none
    oa.step()
    assert float(oa._status[1]) == 1.0                                                              # one step only


# ---- the captured step ------------------------------------------------------------------------------------------------
def _model_l():
    from virconv_b200.backbone import VirConvL8x
    m = VirConvL8x(CFG_L, 8, [1408, 1600, 80], precision='bf16')
    fill_module(m, 666)
    return m.to(DEV).train()


def _model_t():
    from virconv_b200.backbone import VirConv8x
    m = VirConv8x(CFG_T, 8, [1408, 1600, 80], precision='bf16', discard_mode='paper', discard_rng='device')
    fill_module(m, 667)
    return m.to(DEV).train()


def _batch_l(ids, **kw):
    from virconv_b200 import scenes
    b = scenes.make_batch(ids, training=True, **dict(dict(n_lidar=4096, n_virtual=9000, max_voxels=7000), **kw))
    return {'voxel_features': torch.from_numpy(b.voxel_features.copy()).to(DEV),
            'voxel_coords': torch.from_numpy(b.voxel_coords.copy()).to(DEV), 'batch_size': b.batch_size, 'calib': b.calib,
            'aug_param': torch.from_numpy(b.aug_param.copy())}


def _batch_t(ids):
    from virconv_b200 import scenes
    b = scenes.make_batch_mm(ids, max_voxels=3000, training=True, n_lidar=4096, n_virtual=6000)
    bd = {k: torch.from_numpy(v.copy()).to(DEV) for k, v in b.arrays.items()}
    bd.update(batch_size=b.batch_size, calib=b.calib, aug_param=torch.from_numpy(b.aug_param.copy()),
              stvd_seed=torch.tensor([1234], dtype=torch.int64, device=DEV))
    return bd


def _loss(out):
    from virconv_b200.graph import masked_mean
    ts = [out['encoded_spconv_tensor']]
    for g in ('multi_scale_3d_features', 'multi_scale_3d_features_mm'):
        ts += list(out.get(g, {}).values())
    return sum(masked_mean(t) for t in ts)


@pytest.mark.parametrize('which', ['L', 'T'])
def test_captured_step_with_the_update_inside(which):
    """N replays of GraphedStep(optimizer=...) under a OneCycle schedule against N times (GraphedStep, then the eager fused
    step()) from the same state: bit-identical parameters, Adam state and step count, so capture and warm-up applied nothing;
    the torch update of a third copy, fed the same gradients, stays within fp32 rounding."""
    from virconv_b200.graph import GraphedStep
    from virconv_b200.optim import FusedAdamOneCycle
    make_model, make_batch = (_model_l, _batch_l) if which == 'L' else (_model_t, _batch_t)
    batches = [make_batch([1, 2]), make_batch([3, 4])]
    N, wd, max_norm = 5, 0.01, 10.0
    sched = [ooptim.one_cycle(i, N, 0.003, [0.95, 0.85], 10, 0.4) for i in range(N)]
    torch.use_deterministic_algorithms(True)
    try:
        models = [make_model() for _ in range(3)]
        for m in models[1:]:
            m.load_state_dict(models[0].state_dict())
        p_init = [p.detach().clone() for p in models[0].parameters()]
        opts = [FusedAdamOneCycle.from_model(m, wd=wd) for m in models[:2]]
        tgroups, adam = _torch_arm(models[2])
        steps = [GraphedStep(models[0], _loss, margin=1.35, grain=256, optimizer=opts[0], max_grad_norm=max_norm),
                 GraphedStep(models[1], _loss, margin=1.35, grain=256)]
        norms = []
        for i in range(N):
            batch = batches[i % 2]
            lr, mom = sched[i]
            for o in opts:
                o.lr, o.mom = lr, mom
            steps[0](batch)
            steps[1](batch)
            opts[1].step(max_norm=max_norm)
            for p, q in zip(models[1].parameters(), models[2].parameters()):       # the torch arm: the same gradients
                q.grad = None if p.grad is None else p.grad.clone()
            _torch_step(tgroups, adam, lr, mom, wd, max_norm, list(models[2].parameters()))
            torch.cuda.synchronize()
            norms.append(float(opts[0].last_total_norm))
            assert opts[0].applied_steps() == i + 1 == opts[1].applied_steps(), i      # (i = 0: capture and warm-up applied nothing)
            bad = [k for (k, p), q in zip(models[0].named_parameters(), models[1].parameters()) if not torch.equal(p, q)]
            assert not bad, (i, bad[:5])
            assert float(opts[1].last_total_norm) == norms[-1]
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(opts[0].exp_avg_flat, opts[1].exp_avg_flat) and torch.equal(opts[0].exp_avg_sq_flat, opts[1].exp_avg_sq_flat)
    assert opts[0].skipped_steps() == 0 and steps[0].recaptures == 1
    assert steps[0].launches_per_replay == steps[1].launches_per_replay + 2
    assert all(np.isfinite(n) and n > 0 for n in norms), norms
    moved = [not torch.equal(p, q) for p, q in zip(models[0].parameters(), p_init)]
    assert all(moved)
    # the torch arm was fed the same gradients every iteration: the two updates differ by fp32 rounding only
    for (k, p), q in zip(models[0].named_parameters(), models[2].parameters()):
        assert _rel(p, q) < 1e-5, k


def test_recapture_neither_loses_nor_doubles_a_step():
    from virconv_b200.graph import GraphedStep
    from virconv_b200.optim import FusedAdamOneCycle
    small = _batch_l([1, 2], n_lidar=2048, n_virtual=4000, max_voxels=2500)
    large = _batch_l([3, 4])
    model, twin = _model_l(), _model_l()
    opt, ref = FusedAdamOneCycle.from_model(model, wd=0.01), FusedAdamOneCycle.from_model(twin, wd=0.01)
    torch.use_deterministic_algorithms(True)
    try:
        step = GraphedStep(model, _loss, margin=1.2, grain=256, optimizer=opt, max_grad_norm=10.0)
        plain = GraphedStep(twin, _loss, margin=1.2, grain=256)
        calls = 0
        for batch in (small, small, large, small, large):
            step(batch)
            plain(batch)
            ref.step(max_norm=10.0)
            calls += 1
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    assert large['voxel_features'].shape[0] > small['voxel_features'].shape[0] * 1.2 and step.recaptures == 2 == plain.recaptures
    assert opt.applied_steps() + opt.skipped_steps() == calls
    assert opt.applied_steps() == calls and ref.applied_steps() == calls        # the input buffers were the limit: nothing skipped
    assert torch.equal(opt.exp_avg_sq_flat, ref.exp_avg_sq_flat)
    assert all(torch.equal(p, q) for p, q in zip(model.parameters(), twin.parameters()))


def test_pipelined_step_and_world_size_refuse_an_optimizer(monkeypatch):
    from virconv_b200.graph import GraphedStep, PipelinedStep
    from virconv_b200.optim import FusedAdamOneCycle
    model = _model_l()
    opt = FusedAdamOneCycle.from_model(model, wd=0.01)
    with pytest.raises(ValueError, match='PipelinedStep'):
        PipelinedStep(model, _loss, optimizer=opt)
    monkeypatch.setattr(torch.distributed, 'is_initialized', lambda: True)
    monkeypatch.setattr(torch.distributed, 'get_world_size', lambda *a: 2)
    with pytest.raises(ValueError, match='all-reduce'):
        GraphedStep(model, _loss, optimizer=opt)
    GraphedStep(model, _loss)                                       # without an optimizer: as before
