"""CPU: text-line crops.  oracle/crop.py equals cv2.warpAffine with the crop recipe (include/ctpn_b200.h), with IPP on and
off, on random lines, the golden H and O lines, lines partly or wholly outside the image, zero-height lines, the minimum
width, integer and half-pixel corners and crop heights 2, 32 and 256; ctpn_line_crop_widths_host equals the oracle's
widths; ctpn_line_crops_u8 refuses every bad argument with an error naming it, before any CUDA call."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest

from ctpn_b200 import _native as N
from ctpn_b200.engine import check_crop_height
from oracle import crop

HERE = os.path.dirname(os.path.abspath(__file__))


def cv2_crop(im, line, Hc):
    Wc = crop.crop_width(line, Hc)
    return cv2.warpAffine(im, crop.crop_matrix(line, Hc, Wc), (Wc, Hc), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP,
                          borderMode=cv2.BORDER_REPLICATE)


def parallelogram(x1, y1, length, height, angle):
    """An O-mode line: TL, TR = TL + length along angle, BL = TL + height across it, BR = TR + BL - TL."""
    x2, y2 = x1 + length * np.cos(angle), y1 + length * np.sin(angle)
    x3, y3 = x1 - height * np.sin(angle), y1 + height * np.cos(angle)
    return np.array([x1, y1, x2, y2, x3, y3, x2 + x3 - x1, y2 + y3 - y1, 0.95])


def random_cases(seed, n):
    """(canvas, line, Hc): random canvases and lines, a third with integer corners and a fifth with half-pixel ones, some
    of zero height, some partly or wholly outside the canvas."""
    rng = np.random.default_rng(seed)
    out = []
    for t in range(n):
        h, w = (int(v) for v in rng.integers(8, 260, 2))
        im = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        x1, y1 = rng.uniform(-0.3 * w, 1.3 * w), rng.uniform(-0.3 * h, 1.3 * h)
        if t % 3 == 0:
            x1, y1 = np.round(x1), np.round(y1)
        elif t % 5 == 0:
            x1, y1 = np.floor(x1) + 0.5, np.floor(y1) + 0.5
        line = parallelogram(x1, y1, rng.uniform(1, 1.2 * w), 0.0 if t % 11 == 0 else rng.uniform(0.5, 0.4 * h),
                             rng.uniform(-0.4, 0.4))
        if t % 3 == 0:
            line[:8] = np.round(line[:8])
        out.append((im, line, int(rng.choice([2, 32, 48, 256] if t % 8 == 0 else [32, 48]))))
    return out


def golden_lines():
    with np.load(os.path.join(HERE, "golden", "reference_postproc.npz")) as z:
        return {k: z[k] for k in z.files if k.startswith("text_")}


def special_lines():
    """Hand-made lines: horizontal H boxes with integer and half-pixel corners, zero height (ht = 0 -> max(ht, 1)),
    zero length (Wc = 2), a line wholly outside the image, one across its corner, and a vertical one."""
    H = lambda x1, y1, x2, y2: np.array([x1, y1, x2, y1, x1, y2, x2, y2, 0.9])   # noqa: E731
    return [H(10, 12, 90, 40), H(10.5, 12.5, 90.5, 40.5), H(0, 0, 119, 79), H(30, 20, 30, 20), H(40, 33, 70, 33),
            H(-300, -200, -100, -150), H(200, 150, 400, 300), H(-20, -10, 30, 25), parallelogram(50, 5, 60, 30, np.pi / 2),
            parallelogram(3.5, 70.5, 100, 8, -0.6), H(60, 10, 61, 70)]


@pytest.fixture(params=[True, False], ids=["ipp", "noipp"])
def ipp(request):
    before = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(request.param)
    yield request.param
    cv2.ipp.setUseIPP(before)


def test_oracle_equals_cv2_on_random_lines(ipp):
    for i, (im, line, Hc) in enumerate(random_cases(11, 400)):
        got = crop.line_crop(im, line, Hc)
        assert np.array_equal(got, cv2_crop(im, line, Hc)), (i, Hc, line)


@pytest.mark.parametrize("Hc", [2, 32, 256])
def test_oracle_equals_cv2_on_golden_and_special_lines(ipp, Hc):
    rng = np.random.default_rng(Hc)
    for name, lines in sorted(golden_lines().items()):
        right, bottom = lines[:, 0:8:2].max(), lines[:, 1:8:2].max()
        # the canvas stops inside the lines' extent, so that some of them reach past it
        im = rng.integers(0, 256, (int(bottom * 0.9) + 1, int(right * 0.9) + 1, 3), dtype=np.uint8)
        for j, line in enumerate(lines):
            assert np.array_equal(crop.line_crop(im, line, Hc), cv2_crop(im, line, Hc)), (name, j)
    im = rng.integers(0, 256, (80, 120, 3), dtype=np.uint8)
    for j, line in enumerate(special_lines()):
        assert np.array_equal(crop.line_crop(im, line, Hc), cv2_crop(im, line, Hc)), j


def test_width_rule_edges():
    lines = special_lines()
    assert crop.crop_width(lines[3], 32) == 2                       # a point: len 0
    assert crop.crop_width(lines[4], 32) == 32 * 30                 # ht = 0 counts as 1
    assert crop.crop_width(lines[0], 32) == int(np.rint(32 * 80 / 28.0))
    # round half to even: 32 * 5 / 64 = 2.5 -> 2, 32 * 7 / 64 = 3.5 -> 4
    assert crop.crop_width([0, 0, 5, 0, 0, 64], 32) == 2 and crop.crop_width([0, 0, 7, 0, 0, 64], 32) == 4
    padded, widths = crop.line_crops(np.zeros((80, 120, 3), np.uint8), np.stack(lines), 32)
    assert padded.shape == (len(lines), 32, widths.max(), 3)


def host_widths(lines, Hc):
    lines = np.ascontiguousarray(lines, np.float64).reshape(-1, 9)
    w = np.full(len(lines), -7, np.int32)
    rc = N.lib.ctpn_line_crop_widths_host(N.ptr(lines), len(lines), Hc, N.ptr(w))
    return rc, w


@pytest.mark.parametrize("Hc", [2, 32, 256])
def test_host_widths_equal_the_oracle(Hc):
    lines = [ln for _, ln, _ in random_cases(5, 300)] + special_lines()
    lines += [ln for v in golden_lines().values() for ln in v]
    lines = np.stack(lines)
    rc, w = host_widths(lines, Hc)
    assert rc == 0 and np.array_equal(w, crop.crop_widths(lines, Hc))
    assert host_widths(lines[:0], Hc)[0] == 0


def test_host_widths_refuse_what_has_no_width():
    good = special_lines()[0]
    for j, bad in ((1, [np.nan] + [0] * 8), (2, [0, 0, np.inf, 0, 0, 5, 0, 0, 0]), (0, [0, 0, 1e9, 0, 0, 1, 0, 0, 0])):
        lines = np.stack([good] * j + [np.array(bad, np.float64)] + [good])
        rc, _ = host_widths(lines, 32)
        assert rc == N.ERR_INVALID and "line %d:" % j in N.last_error()
    for Hc in (1, 257, 0, -3):
        assert host_widths(good, Hc)[0] == N.ERR_INVALID and "crop height %d" % Hc in N.last_error()
    w = np.zeros(1, np.int32)
    assert N.lib.ctpn_line_crop_widths_host(None, 1, 32, N.ptr(w)) == N.ERR_INVALID and "null" in N.last_error()
    assert N.lib.ctpn_line_crop_widths_host(None, -1, 32, None) == N.ERR_INVALID


# ---- ctpn_line_crops_u8: validation before any CUDA call -------------------------------------------------------------------
# The pointers below are never dereferenced: every call is refused before the library touches the device.
FAKE = 1 << 40


def crops_call(B=3, rows=10, Hc=32, hw=None, num=None, wmax=None, outs=None, canvas=FAKE, lines=FAKE, status=FAKE,
               batch_pitch=None, row_pitch=None, descriptors=True):
    hw = np.array(hw if hw is not None else [[40, 50]] * B, np.int32)
    num = np.array(num if num is not None else [2] * B, np.int32)
    wmax = np.array(wmax if wmax is not None else [64] * B, np.int32)
    outs = np.array(outs if outs is not None else [FAKE + (k << 20) for k in range(B)], np.uint64)
    row_pitch = 50 * 3 if row_pitch is None else row_pitch
    batch_pitch = 40 * row_pitch if batch_pitch is None else batch_pitch
    arrs = (hw, num, wmax, outs) if descriptors else (None,) * 4
    return N.lib.ctpn_line_crops_u8(C.c_void_p(canvas), batch_pitch, row_pitch, N.ptr(arrs[0]), C.c_void_p(lines), B, rows,
                                    Hc, N.ptr(arrs[1]), N.ptr(arrs[2]), N.ptr(arrs[3]), C.c_void_p(status), None)


BAD_CALLS = [
    (dict(descriptors=False), "null descriptor array"),
    (dict(B=0), "batch = 0, must be 1..64"),
    (dict(B=65), "batch = 65, must be 1..64"),
    (dict(Hc=1), "crop height 1, must be 2..256"),
    (dict(Hc=257), "crop height 257, must be 2..256"),
    (dict(rows=-1, num=[0, 0, 0]), "rows = -1"),
    (dict(row_pitch=0), "bad canvas pitches"),
    (dict(num=[2, 11, 2]), "image 1: 11 lines, must be 0..rows = 10"),
    (dict(num=[2, 2, -1]), "image 2: -1 lines"),
    (dict(hw=[[40, 50], [0, 50], [40, 50]]), "image 1: bad size 0 x 50"),
    (dict(hw=[[40, 50], [40, 50], [40, 51]]), "image 2: 40 x 51 x 3 does not fit the canvas pitches"),
    (dict(hw=[[41, 50], [40, 50], [40, 50]]), "image 0: 41 x 50 x 3 does not fit the canvas pitches"),
    (dict(outs=[FAKE, 0, FAKE]), "image 1: null output with 2 lines"),
    (dict(wmax=[64, 64, 1]), "image 2: padded width 1, must be 2..1048576"),
    (dict(wmax=[(1 << 20) + 1, 64, 64]), "image 0: padded width 1048577"),
    (dict(canvas=0), "null canvas, lines or status"),
    (dict(lines=0), "null canvas, lines or status"),
    (dict(status=0), "null canvas, lines or status"),
]


@pytest.mark.parametrize("kwargs,match", BAD_CALLS, ids=[m for _, m in BAD_CALLS])
def test_crops_refuse_bad_arguments(kwargs, match):
    assert crops_call(**kwargs) == N.ERR_INVALID
    assert match in N.last_error(), N.last_error()


def test_crops_without_lines_need_no_output_and_valid_calls_reach_the_device_check():
    """An image without lines needs no output pointer or width; a valid call on a machine without a GPU gets as far as the
    device check (so each refusal above came from its own rule)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("the device check is the GPU-less machine's answer; the GPU tests launch real calls")
    assert crops_call(num=[2, 0, 2], outs=[FAKE, 0, FAKE], wmax=[64, 0, 64]) == N.ERR_NO_DEVICE
    assert crops_call() == N.ERR_NO_DEVICE


@pytest.mark.parametrize("value", [1, 257, 0, 32.0, "32", True])
def test_engine_refuses_a_bad_crop_height(value):
    with pytest.raises(ValueError, match="crop_height must be None or an int 2..256"):
        check_crop_height(value, "detect_lines_images")
    for ok in (None, 2, 32, np.int64(256)):
        check_crop_height(ok, "detect_lines_images")
