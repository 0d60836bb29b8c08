"""CPU tests (no GPU): the drop-in boundary — the C-ABI library builds, loads and exports every symbol the
header declares; the spconv-compatible module surface and the backbone keep the reference's names, shapes
and state_dict layout; the product refuses to run without CUDA (no fallback)."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_builds_loads_and_exports_every_declared_symbol(lib_built):
    from virconv_b200 import _lib
    lib = _lib.load()
    header = open(os.path.join(ROOT, 'include', 'virconv_b200.h')).read()
    header = re.sub(r'/\*.*?\*/', '', header, flags=re.S)
    declared = set(re.findall(r'\b(vc_[a-z0-9_]+)\s*\(', header))
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), f'{name} declared in include/virconv_b200.h but not exported'
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    assert lib.vc_version() >= 100


def test_host_side_entry_points_need_no_gpu(lib_built):
    from virconv_b200 import _lib
    lib = _lib.load()
    o = _lib.host_i32([0, 0, 0])
    assert lib.vc_conv_out_shape(3, _lib.host_i32([81, 1600, 1408]), _lib.host_i32([3, 3, 3]), _lib.host_i32([2, 2, 2]),
                                 _lib.host_i32([1, 1, 1]), _lib.host_i32([1, 1, 1]), o) == 0
    assert list(o) == [41, 800, 704]
    assert lib.vc_subm_rulebook_ws_bytes(1000) == 2048 * 8
    assert lib.vc_conv_ws_bytes(64, 32, 27) == 27 * 64 * 32 * 4
    # error path: message, no exception / exit
    assert lib.vc_conv_out_shape(5, o, o, o, o, o, o) < 0
    assert b'ndim' in lib.vc_last_error()


def test_no_cpu_fallback():
    from virconv_b200 import ops, spconv_compat as sp, _lib
    idx = torch.zeros((4, 4), dtype=torch.int32)
    with pytest.raises(_lib.VirConvLibraryError):
        ops.build_subm_rulebook(idx, 1, [4, 4, 4], 3)
    x = sp.SparseConvTensor(torch.zeros(4, 8), idx, [4, 4, 4], 1)
    with pytest.raises(_lib.VirConvLibraryError):
        sp.SubMConv3d(8, 8, 3, bias=False)(x)
    with pytest.raises(_lib.VirConvLibraryError):
        x.dense()


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, 'virconv_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith('.py'):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle\b', src, flags=re.M), f


def test_spconv_surface_and_state_dict_layout():
    from virconv_b200 import spconv_compat as sp
    from virconv_b200.backbone import VirConvL8x
    cfg = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
    m = VirConvL8x(cfg, 8, np.array([1408, 1600, 80]))
    sd = m.state_dict()
    assert sum(p.numel() for p in m.parameters()) == 425856                     # SURVEY Appendix A.1
    assert sd['vir_conv1.d3_conv1.0.weight'].shape == (8, 3, 3, 3, 8)           # (C_out, kz, ky, kx, C_in)
    assert sd['vir_conv2.down_layer.0.weight'].shape == (32, 3, 3, 3, 16)
    assert sd['vir_conv3.d2_conv2.0.weight'].shape == (32, 3, 3, 32)
    assert sd['conv_out.0.weight'].shape == (64, 3, 1, 1, 64)
    assert 'vir_conv4.d3_conv2.1.running_var' in sd and 'conv_out.1.num_batches_tracked' in sd
    assert m.num_point_features == {'x_conv1': 16, 'x_conv2': 32, 'x_conv3': 64, 'x_conv4': 64}
    assert m.sparse_shape == [81, 1600, 1408]
    # conv modules are leaf modules owning `weight` (optimizer flattening, optimization/__init__.py:26-27)
    for mod in m.modules():
        if isinstance(mod, sp.SparseConvolution):
            assert len(list(mod.children())) == 0 and isinstance(mod.weight, nn.Parameter)
            assert isinstance(mod, sp.conv.SparseConvolution)
    bn = m.vir_conv1.d3_conv1[1]
    assert isinstance(bn, nn.BatchNorm1d) and bn.eps == 1e-3 and bn.momentum == 0.01
    # indice_keys are the reference's (spconv_backbone.py:170,186,192,199,205,564)
    keys = sorted(mod.indice_key for mod in m.modules() if isinstance(mod, sp.SparseConvolution))
    assert 'spvir2' in keys and 'subm1vir1' in keys and 'subm4vir4' in keys and 'spconv_down2' in keys and len(keys) == 20


def test_sparse_conv_tensor_contract():
    from virconv_b200 import spconv_compat as sp
    t = sp.SparseConvTensor(torch.zeros(3, 8), torch.zeros((3, 4), dtype=torch.int32), [4, 5, 6], 1)
    assert 'replace_feature' in t.__dir__()                       # pcdet/utils/spconv_utils.py:59
    with pytest.raises(ValueError):
        t.features = torch.ones(3, 8)                             # spconv 2.x forbids the setter
    u = t.replace_feature(torch.ones(3, 8))
    assert u is not t and u.indices is t.indices and u.indice_dict is t.indice_dict
    t.indices = t.indices[:2]                                     # assignable (spconv_backbone.py:147)
    assert t.indices.shape[0] == 2


def test_install_as_spconv_satisfies_reference_imports():
    import importlib
    import sys
    from virconv_b200 import spconv_compat as sp
    saved = {k: sys.modules.get(k) for k in ('spconv', 'spconv.pytorch', 'spconv.pytorch.conv')}
    try:
        sp.install_as_spconv()
        spconv = importlib.import_module('spconv.pytorch')
        assert spconv.SubMConv3d is sp.SubMConv3d and spconv.conv.SparseConvolution is sp.SparseConvolution
        for name in ('SparseConvTensor', 'SparseSequential', 'SparseConv3d', 'SubMConv2d', 'SparseConv2d',
                     'SparseInverseConv3d', 'SparseModule'):
            assert hasattr(spconv, name)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_projection_params_match_oracle_host_math():
    from virconv_b200 import ops, scenes
    from oracle import index2uv as ouv
    cal = scenes.Calib()
    assert np.array_equal(ops.compose_lidar_to_rect(cal.V2C, cal.R0), ouv.compose_lidar_to_rect(cal.V2C, cal.R0))
    p = ops.projection_params([cal, cal], np.array([[0.3, 1, 0.98], [-0.2, 0, 1.02]], np.float32), 2, 'cpu').numpy()
    assert p.shape == (2, 28) and p[0, 20] == 1 and p[0, 22] == 1 and p[1, 22] == 0
    assert p[0, 23] == np.cos(np.float32(-0.3)) and p[0, 24] == np.sin(np.float32(-0.3))


def test_stvd_keep_rows_follow_reference_rng():
    from virconv_b200.backbone import stvd_keep_rows
    np.random.seed(5)
    want = np.random.permutation(1000)[:int(1000 * (1 - 0.1))]
    np.random.seed(5)
    got = stvd_keep_rows(1000, 0.1)
    assert np.array_equal(got, np.sort(want)) and got.shape[0] == 900


def test_executor_plan_layout_and_host_side_validation(lib_built):
    """The plan a VirConvL8x hands to the native executor: 40 ops (12 rulebook builds, 4 projections, 20 conv+BN+ReLU,
    4 concats), index ops on the side stream, reference indice_keys attached to the rulebooks; a malformed plan is
    rejected on the host before any CUDA call."""
    import ctypes
    import numpy as np
    from virconv_b200 import _lib, executor
    from virconv_b200.backbone import VirConvL8x
    cfg = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
    m = VirConvL8x(cfg, 8, [1408, 1600, 80])
    plan = m._plan()
    oi, of, lf, sizes, offs = plan.finalize()
    assert oi.shape == (40, executor.OPI) and of.shape == (40, executor.OPF) and lf.shape == (20, 2)
    kinds = oi[:, 0].tolist()
    assert (kinds.count(executor.OP_SUBM_RB), kinds.count(executor.OP_CONV_RB), kinds.count(executor.OP_INDEX2UV),
            kinds.count(executor.OP_CBR), kinds.count(executor.OP_CAT)) == (8, 4, 4, 20, 4)
    # feature ops on the main stream (0); strided-conv rulebooks on the index stream (1); submanifold rulebooks + projection on 2
    assert all((oi[i, 1] == 0) == (oi[i, 0] in (executor.OP_CBR, executor.OP_CAT)) for i in range(40))
    assert all(oi[i, 1] == 2 for i in range(40) if oi[i, 0] == executor.OP_INDEX2UV)
    assert all(oi[i, 1] == 2 for i in range(40) if oi[i, 0] == executor.OP_SUBM_RB)
    assert all(oi[i, 1] == 1 for i in range(40) if oi[i, 0] == executor.OP_CONV_RB)
    assert int(offs[-1]) == sum(p.numel() for p in m.parameters())
    assert [n for n, _, _ in plan.published] == ['x_conv1', 'x_conv2', 'x_conv3', 'x_conv4', 'out']
    keys = sorted(k for ks, *_ in plan.rb_keys.values() for k in ks)
    assert keys == sorted(mod.indice_key for mod in m.modules() if hasattr(mod, 'indice_key'))
    assert plan.eligible()
    # every conv's input slot was produced before it is consumed; slot 0 needs no input gradient
    made = {0}
    for r in oi:
        if r[0] == executor.OP_CBR:
            assert r[2] in made and (r[21] == 0) == (r[2] == 0)
            made.add(r[3])
        elif r[0] == executor.OP_CAT:
            assert r[2] in made and r[3] in made
            made.add(r[4])
    lib = _lib.load()
    bad = oi.copy()
    bad[3, 0] = 99
    state = np.zeros(lib.vc_exec_state_bytes(), dtype=np.uint8)
    rc = lib.vc_exec_forward(bad.ctypes.data, of.ctypes.data, 40, None, None, 20, None, 8, None, 1, _lib.host_i32([41, 1600, 1408]),
                             2, None, 1, 0, 1, None, 0, None, None, state.ctypes.data, state.size, None, None, 1, None, None, None, None)
    assert rc == -1 and b'unknown kind' in lib.vc_last_error()
    out = (ctypes.c_longlong * 8)()
    assert lib.vc_exec_query(state.ctypes.data, 0, 0, out) == -1        # not a valid state blob
    assert lib.vc_exec_query(state.ctypes.data, 6, 0, out) == -1        # (the backward operands of a layer, too)


def test_model_with_a_built_plan_can_be_copied_and_pickled():
    """The executor plan is a cache: deepcopy / torch.save of the owning model drop it (it may hold CUDA events) and the
    copy rebuilds its own on first use; state_dict keys are unaffected."""
    import copy
    import io
    import torch
    from virconv_b200.backbone import VirConv8x
    cfg = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.15, NUM_FILTERS=[16, 32, 64, 64], MM=True)
    m = VirConv8x(cfg, 8, [1408, 1600, 80])
    keys = set(m.state_dict())
    m._plan_lidar().inflight[0] = [object()]
    m._plan_mm()
    twin = copy.deepcopy(m)
    assert twin._plan_lidar_cache is None and len(twin._plan_lidar().layers) == 12 and len(twin._plan_mm().layers) == 19
    assert twin._plan_lidar().layers[0][0] is twin.conv_input[0]            # bound to the COPY's modules
    buf = io.BytesIO()
    torch.save(m, buf)
    buf.seek(0)
    again = torch.load(buf, weights_only=False)
    assert again._plan_mm_cache is None and again._plan_mm().eligible()
    assert set(m.state_dict()) == keys == set(again.state_dict())
