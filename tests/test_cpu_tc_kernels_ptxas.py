"""What ptxas makes of the persistent tensor-core kernels, and the shared-memory plan of the conv kernel (host-only).

`tc_conv_persist_kernel` (conv_tc2.cu) and `tc_wgrad_half_kernel` (wgrad_tc3.cu) are compiled with the library's own flags
plus `-Xptxas -v`.  No instantiation may have its wgmma instructions serialized (ptxas warning C7520: the consumer branch
must be provably warp-uniform) or spill to local memory.  Skipped where nvcc is not installed."""
import os
import re
import subprocess
from concurrent.futures import ThreadPoolExecutor

import pytest

from virconv_b200 import build

KERNELS = {'conv_tc2.cu': 'tc_conv_persist_kernel', 'wgrad_tc3.cu': 'tc_wgrad_half_kernel'}
CHANNELS = (16, 32, 64)


def _ptxas_log(src, out_dir):
    path = os.path.join(build.CSRC, src)
    cmd = [build.NVCC] + build.flags_for(path) + ['-Xptxas', '-v', '-c', path, '-o', os.path.join(out_dir, src + '.o')]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r.stdout + r.stderr


def _entries(log, kernel):
    """{mangled name: (stack, spill stores, spill loads)} of every entry function of `kernel` in a ptxas -v log."""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1) if kernel in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            out[cur] = tuple(int(g) for g in m.groups())
            cur = None
    return out


@pytest.fixture(scope='module')
def ptxas_logs(tmp_path_factory):
    if not os.path.exists(build.NVCC):
        pytest.skip('nvcc is not installed')
    d = str(tmp_path_factory.mktemp('ptxas'))
    with ThreadPoolExecutor(max_workers=len(KERNELS)) as ex:
        logs = list(ex.map(lambda s: _ptxas_log(s, d), KERNELS))
    return dict(zip(KERNELS, logs))


@pytest.mark.parametrize('src', sorted(KERNELS))
def test_wgmma_not_serialized(ptxas_logs, src):
    kernel = KERNELS[src]
    bad = [ln for ln in ptxas_logs[src].splitlines() if 'C7520' in ln and kernel in ln]
    assert not bad, '\n'.join(bad)


@pytest.mark.parametrize('src', sorted(KERNELS))
def test_no_local_memory(ptxas_logs, src):
    kernel = KERNELS[src]
    entries = _entries(ptxas_logs[src], kernel)
    assert len(entries) == len(CHANNELS) ** 2, sorted(entries)       # every <C_in, C_out> instantiation was found
    bad = {name: v for name, v in entries.items() if any(v)}
    assert not bad, bad


def _ring_plan(lib, L, cin, cout, K, bn_sums):
    out = L.host_i32([0, 0, 0, 0])
    L.check(lib.vc_conv_tc2_plan(cin, cout, K, bn_sums, out), 'vc_conv_tc2_plan')
    return out[0], bool(out[1]), out[2], out[3]


# (C_in -> C_out at K = 27): (ring stages, weights resident) at two CTAs per SM (106.5 KB of shared memory each), for a launch
# without BatchNorm sums (registers -> global epilogue) and for one with them (half-tile staging buffer)
PLANS_27 = {(16, 16): ((4, True), (3, True)), (16, 32): ((3, True), (2, True)), (16, 64): ((3, False), (2, False)),
            (32, 16): ((3, True), (3, True)), (32, 32): ((3, False), (3, False)), (32, 64): ((3, False), (2, False)),
            (64, 16): ((4, False), (4, False)), (64, 32): ((3, False), (3, False)), (64, 64): ((3, False), (2, False))}


def test_conv_ring_plan(lib_built):
    from virconv_b200 import _lib as L
    lib = L.load()
    L.check(lib.vc_conv_tc2_config(0), 'vc_conv_tc2_config')
    for (cin, cout), plans in PLANS_27.items():
        for bn_sums, (stages, resident) in enumerate(plans):
            S, res, ctas, smem = _ring_plan(lib, L, cin, cout, 27, bn_sums)
            assert (S, res, ctas) == (stages, resident, 2), (cin, cout, bn_sums)
            assert smem <= 227 * 1024 // 2 - 7 * 1024
    assert _ring_plan(lib, L, 8, 16, 27, 0)[:3] == (4, True, 2)          # C = 8 runs padded to 16
    try:
        L.check(lib.vc_conv_tc2_config(1), 'vc_conv_tc2_config')
        S, res, ctas, smem = _ring_plan(lib, L, 64, 64, 27, 0)
        assert ctas == 1 and S >= 2 * PLANS_27[(64, 64)][0][0] and smem <= 227 * 1024 - 8192
    finally:
        L.check(lib.vc_conv_tc2_config(0), 'vc_conv_tc2_config')
    out = L.host_i32([0, 0, 0, 0])
    assert lib.vc_conv_tc2_plan(48, 64, 27, 0, out) != 0
    assert lib.vc_conv_tc2_plan(64, 64, 0, 0, out) != 0
