"""The executor's index orders (vc_set_index_order, VIRCONV_INDEX_ORDER): 0, 1 and 2 are accepted, anything else is refused,
both through the C entry point and through the environment variable read when the library is loaded."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_set_index_order_values():
    from virconv_b200 import _lib
    lib = _lib.load()
    try:
        for mode in (0, 1, 2):
            assert lib.vc_set_index_order(mode) == 0
        for mode in (-1, 3):
            assert lib.vc_set_index_order(mode) != 0
    finally:
        assert lib.vc_set_index_order(2) == 0


def _load_with(value):
    env = dict(os.environ, VIRCONV_INDEX_ORDER=value)
    return subprocess.run([sys.executable, '-c', 'from virconv_b200 import _lib; _lib.load()'], cwd=ROOT, env=env,
                          capture_output=True, text=True)


def test_environment_index_order():
    assert _load_with('2').returncode == 0
    r = _load_with('3')
    assert r.returncode != 0 and 'VIRCONV_INDEX_ORDER must be 0, 1 or 2' in r.stderr
