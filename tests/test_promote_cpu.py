"""CPU: the argument rules of CTPN_F_PROMOTE and the bf16x3p arithmetic mode (CTPN_ARITH_BF16X3P), which the library checks
before any CUDA call, and the command lines of the tools that measure the mode."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest

from ctpn_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F_RELU, F_PROMOTE = 1, 64
FAKE = C.c_void_p(0x1000)        # never dereferenced: the calls fail their argument checks first


@pytest.mark.parametrize("planes", [1, 2])
def test_promote_flag_needs_three_planes(planes):
    rc = N.lib.ctpn_conv3x3(FAKE, FAKE, FAKE, FAKE, 1, 37, 56, 512, 512, 9, planes, F_RELU | F_PROMOTE, None)
    assert rc == 1
    assert "CTPN_F_PROMOTE" in N.last_error()


def test_promote_flag_is_not_a_flag_of_the_f16f8_convolution():
    rc = N.lib.ctpn_conv3x3_f16f8(FAKE, FAKE, FAKE, FAKE, 1, 37, 56, 512, 512, 9, F_RELU | F_PROMOTE, 1.0, 1.0, 1.0, 1.0, None)
    assert rc == 1
    assert "CTPN_F_PROMOTE" in N.last_error()


def test_net_create_accepts_the_promoted_mode():
    h = C.c_void_p()
    assert N.lib.ctpn_net_create(C.byref(h), 5) == 0 and h.value
    assert N.lib.ctpn_net_destroy(h) == 0
    assert N.lib.ctpn_net_create(C.byref(h), 6) == 1


def test_engine_mode_table():
    from ctpn_b200 import Engine
    assert Engine.MODES["bf16x3p"] == 5
    assert Engine.MODES["bf16x3"] == 3 and Engine.MODES["bf16x2"] == 2


@pytest.mark.parametrize("argv", [["tools/head_error_f64.py", "--dry-run", "--modes", "bf16x3p"],
                                  ["tools/time_modes.py", "--dry-run"]])
def test_measurement_tools_parse(argv):
    p = subprocess.run([sys.executable] + argv, cwd=ROOT, capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stderr[-2000:]
    rec = json.loads(p.stdout.strip().splitlines()[-1])
    assert "bf16x3p" in rec["modes"]
