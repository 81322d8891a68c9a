"""CPU: argument checking of the batched device text-line connector (ctpn_text_lines) before any CUDA call, its workspace
size, CTPN_ERR_NO_DEVICE without a GPU, and the demo's --device-lines usage rule."""
import ctypes as C

import numpy as np
import pytest

from ctpn_b200 import _native as N

FAKE = C.c_void_p(0x1000)        # a non-null "device" pointer: validation fails before anything dereferences it


def call(rois=FAKE, counts=FAKE, batch=2, rows=1000, im_hw=None, im_scale=None, oriented=0, cfg9=None, lines=FAKE, num=FAKE,
         status=FAKE, ws=FAKE, ws_bytes=None):
    hw = np.array([[600, 900], [900, 600]], np.int32) if im_hw is None else np.ascontiguousarray(im_hw, np.int32)
    sc = np.array([1.0, 0.8], np.float64) if im_scale is None else np.ascontiguousarray(im_scale, np.float64)
    if ws_bytes is None:
        ws_bytes = N.lib.ctpn_text_lines_workspace_bytes(max(batch, 1), max(rows, 0), 900)
    rc = N.lib.ctpn_text_lines(rois, counts, batch, rows, N.ptr(hw) if hw.size else None, N.ptr(sc) if sc.size else None,
                               oriented, cfg9, lines, num, status, ws, ws_bytes, None)
    return rc, N.last_error()


@pytest.mark.parametrize("name", ["rois", "counts", "lines", "num", "status", "ws"])
def test_null_pointers_are_invalid(name):
    rc, msg = call(**{name: None})
    assert rc == N.ERR_INVALID and "null" in msg


def test_null_host_arrays_are_invalid():
    rc = N.lib.ctpn_text_lines(FAKE, FAKE, 1, 10, None, N.ptr(np.ones(1)), 0, None, FAKE, FAKE, FAKE, FAKE, 1 << 30, None)
    assert rc == N.ERR_INVALID and "null" in N.last_error()
    hw = np.array([[10, 10]], np.int32)
    rc = N.lib.ctpn_text_lines(FAKE, FAKE, 1, 10, N.ptr(hw), None, 0, None, FAKE, FAKE, FAKE, FAKE, 1 << 30, None)
    assert rc == N.ERR_INVALID and "null" in N.last_error()


@pytest.mark.parametrize("kw, text", [
    (dict(batch=0), "batch"), (dict(batch=-3), "batch"), (dict(batch=65), "batch"),
    (dict(rows=-1), "rows"), (dict(rows=65537), "rows"),
    (dict(im_hw=[[600, 900], [0, 600]]), "size"), (dict(im_hw=[[600, -5], [900, 600]]), "size"),
    (dict(im_scale=[1.0, 0.0]), "im_scale"), (dict(im_scale=[-1.0, 1.0]), "im_scale"),
    (dict(im_scale=[1.0, float("nan")]), "im_scale"), (dict(im_scale=[float("inf"), 1.0]), "im_scale"),
    (dict(oriented=2), "oriented"),
])
def test_bad_arguments_are_invalid(kw, text):
    rc, msg = call(**kw)
    assert rc == N.ERR_INVALID and text in msg, msg


def test_too_small_workspace_is_invalid():
    need = N.lib.ctpn_text_lines_workspace_bytes(2, 1000, 900)
    rc, msg = call(ws_bytes=need - 1)
    assert rc == N.ERR_INVALID and "workspace" in msg
    # the workspace follows the widest image of the batch
    rc, msg = call(im_hw=[[600, 2000], [900, 600]], ws_bytes=need)
    assert rc == N.ERR_INVALID and "workspace" in msg


def test_workspace_grows_with_batch_rows_and_width():
    ws = N.lib.ctpn_text_lines_workspace_bytes
    assert ws(0, 1000, 900) == 0 and ws(1, -1, 900) == 0 and ws(1, 1000, 0) == 0
    for b in range(1, 64):
        assert ws(b + 1, 1000, 900) > ws(b, 1000, 900)
    prev = 0
    for rows in list(range(0, 300, 7)) + [1000, 1001, 4096, 65536]:
        assert ws(4, rows, 900) >= prev
        prev = ws(4, rows, 900)
    assert ws(4, 1000, 100000) > ws(4, 1000, 900)
    prev = 0
    for w in (1, 16, 600, 900, 1037, 2600, 10000):
        assert ws(2, 1000, w) >= prev
        prev = ws(2, 1000, w)
    assert ws(1, 1000, 900) >= 1000 * 16 * 8          # the NMS bitmask: rows x rows / 64 words


def test_valid_call_without_a_device_is_no_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("this check is for a machine without a GPU")
    rc, msg = call()
    assert rc == N.ERR_NO_DEVICE, msg


def test_demo_device_lines_needs_device_frontend():
    from ctpn import demo
    with pytest.raises(SystemExit):
        demo.main(["--batch", "4", "--device-lines"])
