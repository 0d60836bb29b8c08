"""CPU tests of SyncBatchNorm on the fast path (sync_bn): plan eligibility with converted layers at world size 1 and above
(a fake process group), refusal of mixed groups, the exchange-slot layout, and how the reducer is chosen."""
import copy

import pytest
import torch
import torch.distributed as dist

CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG8 = dict(CFG, MM=True)


def _models():
    from virconv_b200.backbone import VirConv8x, VirConvL8x
    return [VirConvL8x(CFG, 8, [1408, 1600, 80]).train(), VirConv8x(CFG8, 8, [1408, 1600, 80]).train()]


def _plans(m):
    from virconv_b200.backbone import VirConvL8x
    return [m._plan()] if isinstance(m, VirConvL8x) else [m._plan_lidar(), m._plan_mm()]


@pytest.fixture
def fake_world(monkeypatch):
    """torch.distributed as if initialised with `size[0]` ranks (every group)."""
    size = [2]
    monkeypatch.setattr(dist, 'is_available', lambda: True)
    monkeypatch.setattr(dist, 'is_initialized', lambda: True)
    monkeypatch.setattr(dist, 'get_world_size', lambda group=None: size[0])
    return size


@pytest.mark.parametrize('world', [1, 2, 8])
def test_converted_plans_are_eligible(fake_world, world):
    fake_world[0] = world
    from virconv_b200 import sync_bn
    for m in _models():
        conv = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(m))
        for plan in _plans(conv):
            bns = [bn for _, bn in plan.layers]
            assert all(type(bn) is torch.nn.SyncBatchNorm for bn in bns)
            assert plan.eligible()
            assert sync_bn.world_size(bns) == world
            assert sync_bn.active(conv, bns) == (world > 1)
        for plan in _plans(m):                 # the BatchNorm1d model never exchanges
            assert plan.eligible() and not sync_bn.active(m, [bn for _, bn in plan.layers])


def test_world_size_one_without_a_process_group():
    from virconv_b200 import sync_bn
    m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_models()[0])
    bns = [bn for _, bn in m._plan().layers]
    assert not dist.is_initialized()
    assert sync_bn.world_size(bns) == 1 and sync_bn.reducer_for(m, bns) is None


def test_mixed_process_groups_are_refused(fake_world):
    from virconv_b200 import sync_bn
    from virconv_b200.backbone import _module_path_reason
    m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_models()[0], process_group=object())
    plan = m._plan()
    plan.layers[3][1].process_group = object()
    bns = [bn for _, bn in plan.layers]
    with pytest.raises(ValueError, match='process groups'):
        sync_bn.group_of(bns)
    assert not plan.eligible()
    feats = torch.zeros(4, 8)
    assert _module_path_reason(feats, plan) is not None
    # (every rank takes the module path for this reason: torch's SyncBatchNorm exchanges there, nothing raises)
    m._no_module_path_under_sync(plan, _module_path_reason(feats, plan))


@pytest.mark.parametrize('why', ['no input voxels', 'gradient into the voxel features',
                                 'BatchNorm layers in mixed train / eval modes'])
def test_rank_dependent_fallback_raises(fake_world, why):
    """A reason that depends on one rank's batch raises under an active exchange instead of taking the module path (the
    other ranks would wait for its exchanges); a configuration-wide reason does not."""
    from virconv_b200 import backbone
    m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_models()[0])
    plan = m._plan()
    assert why in backbone._RANK_DEPENDENT
    with pytest.raises(RuntimeError, match='SyncBatchNorm across ranks'):
        m._no_module_path_under_sync(plan, why)
    m._no_module_path_under_sync(plan, 'VIRCONV_EXECUTOR=0')
    fake_world[0] = 1
    m._no_module_path_under_sync(plan, why)          # world size 1, no hook: plain BatchNorm, no exchange to keep in step


def test_some_layers_sync_is_refused():
    from virconv_b200 import sync_bn
    m = _models()[0]
    plan = m._plan()
    conv, bn = plan.layers[0]
    sync = torch.nn.SyncBatchNorm(bn.num_features, eps=bn.eps, momentum=bn.momentum)
    plan.layers[0] = (conv, sync)
    with pytest.raises(ValueError, match='of one plan are SyncBatchNorm'):
        sync_bn.group_of([b for _, b in plan.layers])
    assert not plan.eligible()


def test_exchange_slot_layout():
    """Per layer in plan order: forward slot [sum x (C), sum x^2 (C), rows], then backward slot [sum g (C), sum g*xhat (C)]."""
    for m in _models():
        for plan in _plans(m):
            off, total = plan.sync_slots()
            assert off.dtype.name == 'int64' and off.shape == (len(plan.layers), 2) and off.flags['C_CONTIGUOUS']
            pos = 0
            for i, (conv, _) in enumerate(plan.layers):
                c = conv.out_channels
                assert off[i, 0] == pos and off[i, 1] == pos + 2 * c + 1
                pos += 4 * c + 1
            assert total == pos
    plan = _models()[0]._plan()
    assert [plan.layers[i][0].out_channels for i in range(2)] == [8, 8]      # vir_conv1's first two layers (C = 8)
    assert plan.sync_slots()[0][:2].tolist() == [[0, 17], [33, 50]]


def test_reducer_comes_from_the_group_and_the_hook_overrides_it(fake_world, monkeypatch):
    from virconv_b200 import sync_bn
    calls = []
    monkeypatch.setattr(dist, 'all_reduce', lambda t, group=None: calls.append(group))
    group = object()
    m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_models()[0], process_group=group)
    bns = [bn for _, bn in m._plan().layers]
    red = sync_bn.reducer_for(m, bns)
    red(torch.zeros(3), ('', 0, 'forward'))
    assert calls == [group]
    hook = lambda slot, key: None  # noqa: E731
    m.bn_reducer = hook
    assert sync_bn.reducer_for(m, bns) is hook
    fake_world[0] = 1
    assert sync_bn.reducer_for(m, bns) is hook          # the hook forces the exchange at world size 1
    m.bn_reducer = None
    assert sync_bn.reducer_for(m, bns) is None
    m.eval()
    fake_world[0] = 2
    assert sync_bn.reducer_for(m, bns) is None           # eval: the running statistics, nothing exchanged


def test_voxel_pool_reducer(fake_world):
    from virconv_b200 import sync_bn
    from virconv_b200.voxel_pool import NeighborVoxelSAModuleMSG
    mod = NeighborVoxelSAModuleMSG(query_ranges=[[2, 2, 2]], radii=[0.4], nsamples=[16], mlps=[[64, 32, 32]]).train()
    assert sync_bn.reducer_for(mod, [mod.mlps_pos[0][1]]) is None
    mod = torch.nn.SyncBatchNorm.convert_sync_batchnorm(mod)
    assert isinstance(mod.mlps_pos[0][1], torch.nn.SyncBatchNorm)
    assert sync_bn.reducer_for(mod, [mod.mlps_pos[0][1]]) is not None


def test_pipelined_step_refuses_sync_bn_across_ranks(fake_world):
    from virconv_b200.graph import PipelinedStep
    m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_models()[0])
    with pytest.raises(ValueError, match='SyncBatchNorm'):
        PipelinedStep(m, lambda out: None)
