"""CPU tests (no GPU) of the fused parameter update's host side: the float64 restatement against what the reference's own
OptimWrapper + OneCycle + clip_grad_norm_ computed (tests/golden/optim_ref.npz), the parameter groups, the schedule, the
checkpoint layout through a real torch.optim.Adam, the C ABI, and the reference_env binding."""
import os
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'optim_ref.npz')


def _rel(got, want):
    want = np.asarray(want, dtype=np.float64)
    return float(np.abs(np.asarray(got, dtype=np.float64) - want).max() / max(np.abs(want).max(), 1e-30))


def _oracle_run(gold, steps):
    """The float64 restatement over the golden tree, gradients and schedule -> (oracle, names, total norms)."""
    from oracle import optim as ooptim
    from oracle import optim_golden as og
    model = og.golden_tree()
    names = [str(n) for n in list(gold['group0']) + list(gold['group1'])]
    o = ooptim.AdamOneCycle([gold['init.' + n] for n in names], wd=og.CFG['WEIGHT_DECAY'])
    norms = []
    for it in range(steps):
        g = og.golden_grads(model, it)
        o.step([g.get(n) for n in names], float(gold['lr'][it]), float(gold['mom'][it]), og.MAX_NORM,
               norm_only=[v for n, v in g.items() if n not in names])
        norms.append(o.total_norm)
    return o, names, norms


def test_oracle_matches_the_reference_run():
    """Float64 against the reference's float32 run: what separates them after 40 steps is fp32 rounding in the reference's
    own arithmetic, 1e-6 of the largest value of a tensor; the total norms agree to fp32 resolution."""
    from oracle import optim_golden as og
    gold = np.load(GOLDEN)
    for k in og.CHECKPOINTS:
        o, names, norms = _oracle_run(gold, k)
        assert o.t == k and o.skipped == 0
        for i, n in enumerate(names):
            assert _rel(o.p[i], gold['p.%d.%s' % (k, n)]) < 1e-6, (k, n)
            if n.startswith('unused.'):
                assert 'm.%d.%s' % (k, n) not in gold and not o.m[i].any()       # decayed only: no Adam state either side
                continue
            assert _rel(o.m[i], gold['m.%d.%s' % (k, n)]) < 2e-6, (k, n)
            assert _rel(o.v[i], gold['v.%d.%s' % (k, n)]) < 2e-6, (k, n)
    assert _rel(norms, gold['total_norm']) < 1e-6
    assert (gold['total_norm'] > og.MAX_NORM).any() and (gold['total_norm'] < og.MAX_NORM).any()
    # the parent-owned tensor and the frozen one were never updated
    assert np.array_equal(gold['p.40.block.scale'], gold['init.block.scale'])
    assert np.array_equal(gold['p.40.frozen.weight'], gold['init.frozen.weight'])


def test_oracle_skip_rule_and_decay_only():
    from oracle import optim as ooptim
    o = ooptim.AdamOneCycle([np.ones(3), np.full(2, 2.0)], wd=0.1)
    assert not o.step([np.array([1.0, np.inf, 0.0]), None], 0.01, 0.9, 10.0)
    assert not o.step([np.array([1.0, np.nan, 0.0]), None], 0.01, 0.9, 10.0)
    assert not o.step([np.ones(3), None], 0.01, 0.9, 10.0, guard=3)
    assert (o.t, o.skipped) == (0, 3) and np.array_equal(o.p[0], np.ones(3)) and not o.m[0].any()
    assert o.step([np.ones(3), None], 0.01, 0.9, None)
    assert o.t == 1 and o.clip_coef == 1.0
    assert np.allclose(o.p[1], 2.0 * (1 - 0.1 * 0.01), rtol=0, atol=1e-15) and not o.m[1].any()
    # first Adam step: m / (1 - beta1) = g, sqrt(v / (1 - beta2)) = |g| -> p moves by lr * sign(g) (up to eps)
    assert np.allclose(o.p[0], (1 - 0.1 * 0.01) - 0.01, rtol=0, atol=1e-9)


def test_groups_follow_the_reference_rule():
    from oracle import optim_golden as og
    from virconv_b200.optim import leaf_param_groups
    gold = np.load(GOLDEN)
    model = og.golden_tree()
    name_of = {id(p): n for n, p in model.named_parameters()}
    groups, rest = leaf_param_groups(model)
    assert [name_of[id(p)] for p in groups[0]] == [str(n) for n in gold['group0']]
    assert [name_of[id(p)] for p in groups[1]] == [str(n) for n in gold['group1']]
    assert [name_of[id(p)] for p in rest] == ['block.scale']                   # owned by a module with children
    assert 'frozen.weight' not in {name_of[id(p)] for g in groups for p in g}


def test_one_cycle_sequence():
    from oracle import optim as ooptim
    from oracle import optim_golden as og
    gold = np.load(GOLDEN)
    c = og.CFG
    seq = [ooptim.one_cycle(i, og.STEPS, c['LR'], c['MOMS'], c['DIV_FACTOR'], c['PCT_START']) for i in range(og.STEPS)]
    assert np.allclose([s[0] for s in seq], gold['lr'], rtol=1e-14, atol=0)
    assert np.allclose([s[1] for s in seq], gold['mom'], rtol=1e-14, atol=0)
    assert np.argmax(gold['lr']) == int(og.STEPS * c['PCT_START']) and np.argmin(gold['mom']) == np.argmax(gold['lr'])


def test_state_dict_layout_through_torch_adam():
    """pack_state_dict writes what torch.optim.Adam reads and unpack_state_dict reads what it writes; the layout is the one
    the reference's checkpoint holds (two groups, consecutive ids, no entry for a tensor that never had a gradient)."""
    from oracle import optim_golden as og
    from virconv_b200.optim import leaf_param_groups, pack_state_dict, unpack_state_dict
    gold = np.load(GOLDEN)
    o, names, _ = _oracle_run(gold, og.STEPS)
    model = og.golden_tree()
    groups, _ = leaf_param_groups(model)
    hyper = dict(lr=float(gold['lr'][-1]), betas=(float(gold['mom'][-1]), 0.99), eps=1e-8, weight_decay=0, amsgrad=False)
    entries = {i: (torch.from_numpy(o.m[i]).float(), torch.from_numpy(o.v[i]).float())
               for i, n in enumerate(names) if not n.startswith('unused.')}
    sd = pack_state_dict([dict(hyper, params=g) for g in groups], og.STEPS, entries)
    assert sorted(sd['state']) == gold['sd_state_keys'].tolist()
    assert sd['param_groups'][0]['params'] == gold['sd_group0'].tolist()
    assert sd['param_groups'][1]['params'] == gold['sd_group1'].tolist()
    assert sorted(sd['state'][0]) == [str(s) for s in gold['sd_state_fields']]
    assert {float(s['step']) for s in sd['state'].values()} == set(gold['sd_steps'].tolist())
    assert sd['param_groups'][0]['weight_decay'] == int(gold['sd_weight_decay'])

    # into a real Adam over the same groups, one more step there, against one more oracle step
    with torch.no_grad():
        for i, n in enumerate(names):
            dict(model.named_parameters())[n].copy_(torch.from_numpy(o.p[i]).float())
    adam = torch.optim.Adam([{'params': g, 'lr': 0} for g in groups], betas=(0.9, 0.99))
    adam.load_state_dict(sd)
    named = dict(model.named_parameters())
    g = og.golden_grads(model, og.STEPS)
    for n, v in g.items():
        named[n].grad = torch.from_numpy(v.copy())
    named['block.scale'].grad = None
    lr, mom = hyper['lr'], hyper['betas'][0]
    adam.step()
    o.wd = 0.0
    o.step([g.get(n) for n in names], lr, mom, None)
    for i, n in enumerate(names):
        assert _rel(named[n].detach().numpy(), o.p[i]) < 1e-6, n
    # and back
    t, back, g0 = unpack_state_dict(adam.state_dict(), [len(g) for g in groups])
    assert t == og.STEPS + 1 and sorted(back) == sorted(entries) and g0['betas'][0] == mom
    for i in back:
        assert _rel(back[i][0].numpy(), o.m[i]) < 2e-6
    with pytest.raises(ValueError, match='groups'):
        unpack_state_dict(adam.state_dict(), [3, 4])
    bad = adam.state_dict()
    bad['state'][0]['step'] = torch.tensor(3.0)
    with pytest.raises(ValueError, match='step counts'):
        unpack_state_dict(bad, [len(g) for g in groups])


def test_chunk_list():
    from virconv_b200 import optim
    c = optim.chunk_list([1, 4096, 4097, 0, 10000])
    assert c.dtype.itemsize == 16
    assert c['seg'].tolist() == [0, 1, 2, 2, 4, 4, 4]
    assert c['len'].tolist() == [1, 4096, 4096, 1, 4096, 4096, 1808]
    assert c['off'].tolist() == [0, 0, 0, 4096, 0, 4096, 8192]
    assert all(o % 4 == 0 for o in c['off'])


def test_c_abi_symbols(lib_built):
    from virconv_b200 import _lib, optim
    header = open(os.path.join(ROOT, 'include', 'virconv_b200.h')).read()
    lib = _lib.load()
    for sym in ('vc_optim_ws_bytes', 'vc_optim_step'):
        assert sym in _lib.SIGNATURES and sym in header and hasattr(lib, sym)
    assert '#define VC_OPTIM_CHUNK %d' % optim.CHUNK in header and '#define VC_OPTIM_MAX_GUARDS %d' % optim.MAX_GUARDS in header
    assert lib.vc_optim_ws_bytes(0) == 256 and lib.vc_optim_ws_bytes(100) == 256 + 800
    # host-side validation: message, no CUDA call
    assert lib.vc_optim_step(None, 1, None, 1, 1.0, None, 0, None, None, None, 0, None, 0, None) < 0
    assert b'optim' in lib.vc_last_error()


def test_no_cpu_fallback():
    from virconv_b200.optim import FusedAdamOneCycle
    with pytest.raises(ValueError, match='CUDA'):
        FusedAdamOneCycle([torch.nn.Parameter(torch.zeros(4))])


def test_reference_env_flag_binds_the_two_names_only():
    import virconv_b200.reference_env as renv
    saved = {k: sys.modules.get(k) for k in ('train_utils', 'train_utils.optimization', 'train_utils.train_utils')}

    def reference_build(model, cfg):
        return ('reference', cfg.OPTIMIZER)

    def other():
        pass
    try:
        pkg = types.ModuleType('train_utils')
        pkg.__path__ = []
        om = types.ModuleType('train_utils.optimization')
        om.build_optimizer, om.build_scheduler = reference_build, other
        tm = types.ModuleType('train_utils.train_utils')
        tm.clip_grad_norm_, tm.train_one_epoch = torch.nn.utils.clip_grad_norm_, other
        sys.modules.update({'train_utils': pkg, 'train_utils.optimization': om, 'train_utils.train_utils': tm})
        renv.install()
        assert om.build_optimizer is reference_build and tm.clip_grad_norm_ is torch.nn.utils.clip_grad_norm_     # flag off
        renv.install(use_fused_optimizer=True)
        renv.install(use_fused_optimizer=True)                                                                    # (idempotent)
        assert om.build_optimizer._reference is reference_build and om.build_scheduler is other
        assert tm.clip_grad_norm_ is renv._fused_clip_grad_norm_ and tm.train_one_epoch is other
        # other OPTIMIZER values go to the reference's function
        assert om.build_optimizer(None, renv.EasyDict(OPTIMIZER='sgd')) == ('reference', 'sgd')
        # parameters no fused optimizer owns go to torch's clip_grad_norm_
        p = torch.nn.Parameter(torch.ones(4))
        p.grad = torch.full((4,), 3.0)
        norm = tm.clip_grad_norm_([p], 3.0)
        assert abs(float(norm) - 6.0) < 1e-6 and torch.allclose(p.grad, torch.full((4,), 1.5), atol=1e-5)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
