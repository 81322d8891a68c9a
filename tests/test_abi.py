"""CPU: the C-ABI library loads without a GPU and exports every symbol the header declares;
the ctypes table in ctpn_b200/_native.py covers exactly the header."""
import os
import re

import pytest

from ctpn_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "ctpn_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ctpn_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported():
    names = header_functions()
    assert len(names) >= 18
    for n in names:
        assert hasattr(N.lib, n), "libctpn_b200.so does not export %s" % n


def test_ctypes_table_matches_header():
    assert sorted(N.SIGNATURES) == header_functions()


def test_product_library_has_no_test_only_symbols_and_debug_library_has_them():
    """Probes, SIMT reference kernels and ablation switches live in tests/_native/libctpn_b200_dbg.so
    (csrc/testing/ctpn_b200_testing.h), not in the shipped library or the public header."""
    import ctypes as C
    hdr = open(os.path.join(ROOT, "text-detection-ctpn_b200", "csrc", "testing", "ctpn_b200_testing.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    test_only = sorted(set(re.findall(r"\b(ctpn_[a-z0-9_]+)\s*\(", hdr)))
    assert sorted(N.TESTING_SIGNATURES) == test_only and len(test_only) >= 3
    dbg = C.CDLL(os.path.join(ROOT, "tests", "_native", "libctpn_b200_dbg.so"))
    for n in test_only:
        assert not hasattr(N.lib, n), "product library exports test-only symbol %s" % n
        assert hasattr(dbg, n)
    for n in header_functions():
        assert hasattr(dbg, n)


def test_version_and_error_string():
    assert N.lib.ctpn_version() >= 100
    assert isinstance(N.last_error(), str)


def test_invalid_arguments_are_reported_not_crashed():
    # argument validation happens before any CUDA call, so this works without a GPU
    import ctypes as C
    num = C.c_int(-1)
    rc = N.lib.ctpn_nms_host(None, C.byref(num), None, 5, 5, 0.7, 0)
    assert rc == 1 and "null" in N.last_error()
    keep = (C.c_int * 4)()
    rc = N.lib.ctpn_nms_host(keep, C.byref(num), None, 0, 5, 0.7, 0)      # empty input: OK, zero kept
    assert rc == 0 and num.value == 0
    boxes = (C.c_float * 12)()
    rc = N.lib.ctpn_nms_host(keep, C.byref(num), boxes, 4, 3, 0.7, 0)
    assert rc == 1 and "boxes_dim" in N.last_error()
    fh, fw = C.c_int(), C.c_int()
    assert N.lib.ctpn_net_feature_hw(600, 900, C.byref(fh), C.byref(fw)) == 0 and (fh.value, fw.value) == (37, 56)
    assert N.lib.ctpn_net_feature_hw(1200, 1600, C.byref(fh), C.byref(fw)) == 0 and (fh.value, fw.value) == (75, 100)
    assert N.lib.ctpn_conv3x3(None, None, None, None, 1, 8, 8, 64, 64, 9, 1, 0, None) == 1
    assert N.lib.ctpn_nms_workspace_bytes(1, 12000) == 12000 * 188 * 8


def test_product_refuses_to_run_without_a_gpu_or_without_the_library():
    """No CPU fallback anywhere on the product path: without a CUDA device the engine raises and device entry
    points return CTPN_ERR_NO_DEVICE; without the shared library the package does not import."""
    import ctypes as C
    import subprocess
    import sys
    import torch
    if torch.cuda.is_available():
        pytest.skip("this check is for the GPU-less build container")
    from ctpn_b200 import CtpnError, Engine
    with pytest.raises(CtpnError, match="no CPU fallback"):
        Engine(None)
    keep, num, boxes = (C.c_int * 4)(), C.c_int(), (C.c_float * 20)()
    assert N.lib.ctpn_nms_host(keep, C.byref(num), boxes, 4, 5, 0.7, 0) == N.ERR_NO_DEVICE
    with pytest.raises(CtpnError):
        N.check(N.lib.ctpn_device_ok(0), "ctpn_device_ok")
    # a package copy without the .so must fail at import, not fall back
    code = ("import sys, os, shutil, tempfile\n"
            "d = tempfile.mkdtemp()\n"
            "shutil.copytree(%r, os.path.join(d, 'ctpn_b200'), ignore=shutil.ignore_patterns('*.so', '__pycache__'))\n"
            "sys.path.insert(0, d)\n"
            "try:\n"
            "    import ctpn_b200\n"
            "except ImportError as e:\n"
            "    assert 'no CPU fallback' in str(e), e\n"
            "    print('refused')\n"
            "finally:\n"
            "    shutil.rmtree(d)\n") % os.path.dirname(N.__file__)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.stdout.strip() == "refused", out.stdout + out.stderr
