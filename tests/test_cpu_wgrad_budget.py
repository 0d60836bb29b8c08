"""vc_wgrad_launch_geometry (host-only) for every layer of VirConv-L's and VirConv-T's plans: the CTA cap of a weight-gradient
launch holds over all its passes, every pass keeps at least one CTA, and each pass gets an equal share of the cap."""
import math

import pytest

CFG = dict(RETURN_NUM_FEATURES_AS_DICT=True, OUT_FEATURES=64, LAYER_DISCARD_RATE=0.1, NUM_FILTERS=[16, 32, 64, 64])
CFG_T = dict(CFG, LAYER_DISCARD_RATE=0.15, MM=True)


def _plan_layers():
    from virconv_b200.backbone import VirConv8x, VirConvL8x
    ml = VirConvL8x(CFG, 8, [1408, 1600, 80], precision='bf16')
    mt = VirConv8x(CFG_T, 8, [1408, 1600, 80], precision='bf16')
    plans = {'L': [ml._plan()], 'T': [mt._plan_lidar(), mt._plan_mm()]}
    out = []
    for model, ps in plans.items():
        for p in ps:
            for conv, _ in p.layers:
                out.append((model, conv.in_channels, conv.out_channels, math.prod(conv.kernel_size)))
    return out


def _passes(cin, cout, K):
    pad = lambda c: max(16, c)          # noqa: E731  (C = 8 runs padded to 16)
    groups = -(-K // (128 // pad(cin)))
    return -(-groups // (64 // pad(cout)))


def test_geometry_of_every_plan_layer(lib_built):
    from virconv_b200 import _lib as L
    lib = L.load()
    layers = _plan_layers()
    assert {m for m, *_ in layers} == {'L', 'T'}
    out = L.host_i32([0, 0])
    multi = 0
    for model, cin, cout, K in layers:
        for n in (1, 129, 40000, 250000):
            for cap in (1, 7, 33, 66, 99, 132):
                L.check(lib.vc_wgrad_launch_geometry(cin, cout, K, n, cap, out), 'vc_wgrad_launch_geometry')
                gx, passes = out[0], out[1]
                assert passes == _passes(cin, cout, K), (model, cin, cout, K)
                assert gx == max(1, min(-(-n // 128), cap // passes)), (model, cin, cout, K, n, cap)
                if passes <= cap:
                    assert gx * passes <= cap
        multi += _passes(cin, cout, K) > 1
    assert multi > 0


@pytest.mark.parametrize('args', [(8, 16, 27, 0, 66), (64, 64, 27, 100, 0), (48, 64, 27, 100, 66), (64, 64, 0, 100, 66),
                                  (64, 64, 27, -1, 66)])
def test_geometry_rejects_bad_arguments(lib_built, args):
    from virconv_b200 import _lib as L
    lib = L.load()
    out = L.host_i32([7, 7])
    if args[3] == 0:        # no rows: nothing is launched
        assert lib.vc_wgrad_launch_geometry(*args, out) == 0 and out[0] == 0 and out[1] >= 1
    else:
        assert lib.vc_wgrad_launch_geometry(*args, out) != 0
