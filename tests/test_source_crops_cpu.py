"""CPU: line crops out of the source images (crop_from="source").  The crop recipe on the source line lines[:8] / f equals
cv2.warpAffine of the source image at camera sizes, with IPP on and off; ctpn_line_crops_strided_u8 and
ctpn_line_crops_yuv420_u8 refuse every bad argument with an error naming it, before any CUDA call, and valid calls reach
the device check; the engine checks crop_from; a stream of host photos with source crops uploads them whole."""
import ctypes as C

import cv2
import numpy as np
import pytest

from ctpn_b200 import _native as N
from ctpn_b200.engine import check_crop_from, frontend_plan, stream_layout
from oracle import crop

# camera photos (landscape and portrait), a 4K frame, a 3:1 photo and an upscaled 480 x 640
SOURCE_SIZES = [(3024, 4032), (4032, 3024), (2160, 3840), (1000, 3000), (480, 640)]


def source_line(line, f):
    """The source line of a line of the resize_im frame: its corners divided by f in float64 (the score is kept)."""
    src = np.array(line, np.float64)
    src[:8] /= np.float64(f)
    return src


def cv2_crop(im, line, Hc):
    Wc = crop.crop_width(line, Hc)
    return cv2.warpAffine(im, crop.crop_matrix(line, Hc, Wc), (Wc, Hc), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP,
                          borderMode=cv2.BORDER_REPLICATE)


def resized_lines(rng, rh, rw, n):
    """n lines of the resize_im frame (rh x rw): oriented parallelograms, some partly outside the frame, one of height 0,
    some with half-pixel corners."""
    out = []
    for j in range(n):
        x1, y1 = rng.uniform(-0.1 * rw, rw), rng.uniform(-0.1 * rh, rh)
        if j % 4 == 1:
            x1, y1 = np.floor(x1) + 0.5, np.floor(y1) + 0.5
        a, L = rng.uniform(-0.4, 0.4), rng.uniform(5, rw)
        H = 0.0 if j == 2 else rng.uniform(0.5, 60)
        x2, y2, x3, y3 = x1 + L * np.cos(a), y1 + L * np.sin(a), x1 - H * np.sin(a), y1 + H * np.cos(a)
        out.append(np.array([x1, y1, x2, y2, x3, y3, x2 + x3 - x1, y2 + y3 - y1, 0.9]))
    return out


@pytest.mark.parametrize("h,w", SOURCE_SIZES, ids=["%dx%d" % s for s in SOURCE_SIZES])
def test_oracle_on_source_lines_equals_cv2_at_camera_sizes(h, w):
    rng = np.random.default_rng(h * 7 + w)
    im = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    p = frontend_plan([(h, w)])[0]
    before = cv2.ipp.useIPP()
    try:
        for j, line in enumerate(resized_lines(rng, p.resized[0], p.resized[1], 6)):
            src = source_line(line, p.f)
            for Hc in (32, 256):
                got = crop.line_crop(im, src, Hc)
                for ipp in (True, False):
                    cv2.ipp.setUseIPP(ipp)
                    assert np.array_equal(got, cv2_crop(im, src, Hc)), (j, Hc, ipp)
    finally:
        cv2.ipp.setUseIPP(before)


def test_source_widths_are_the_host_widths_of_the_divided_lines():
    """The engine sizes source crops with ctpn_line_crop_widths_host on lines / f divided in numpy: the oracle's widths."""
    rng = np.random.default_rng(4)
    p = frontend_plan([(3024, 4032)])[0]
    lines = np.stack([source_line(ln, p.f) for ln in resized_lines(rng, *p.resized, 40)])
    w = np.zeros(len(lines), np.int32)
    assert N.lib.ctpn_line_crop_widths_host(N.ptr(lines), len(lines), 48, N.ptr(w)) == 0
    assert np.array_equal(w, crop.crop_widths(lines, 48))
    assert (w > crop.crop_widths(np.stack(resized_lines(np.random.default_rng(4), *p.resized, 40)), 48)).any()


# ---- validation before any CUDA call ------------------------------------------------------------------------------------
# The pointers below are never dereferenced: every call is refused before the library touches the device.
FAKE = 1 << 40


def strided_call(B=3, rows=10, Hc=32, hw=None, f=None, num=None, wmax=None, outs=None, srcs=None, nbytes=None, offs=None,
                 strides=None, lines=FAKE, status=FAKE, descriptors=True):
    """B 40 x 50 BGR images, each in a 6000-byte allocation of its own, row stride 150."""
    hw = np.array(hw if hw is not None else [[40, 50]] * B, np.int32)
    f = np.array(f if f is not None else [0.5] * B, np.float64)
    num = np.array(num if num is not None else [2] * B, np.int32)
    wmax = np.array(wmax if wmax is not None else [64] * B, np.int32)
    outs = np.array(outs if outs is not None else [FAKE + (k << 20) for k in range(B)], np.uint64)
    srcs = np.array(srcs if srcs is not None else [FAKE + (k << 24) for k in range(B)], np.uint64)
    nbytes = np.array(nbytes if nbytes is not None else [6000] * B, np.uint64)
    offs = np.array(offs if offs is not None else [0] * B, np.int64)
    strides = np.array(strides if strides is not None else [[150, 3, 1]] * B, np.int64)
    arrs = (srcs, nbytes, offs, strides, hw, f, num, wmax, outs) if descriptors else (None,) * 9
    return N.lib.ctpn_line_crops_strided_u8(*(N.ptr(a) for a in arrs[:6]), C.c_void_p(lines), B, rows, Hc,
                                            *(N.ptr(a) for a in arrs[6:]), C.c_void_p(status), None)


def yuv_call(B=3, rows=10, Hc=32, hw=None, f=None, num=None, wmax=None, outs=None, planes=None, nbytes=None, offs=None,
             strides=None, lines=FAKE, status=FAKE, descriptors=True):
    """B 40 x 50 I420 frames, each plane in an allocation of its own: Y 2000 bytes at pitch 50, U and V 500 at pitch 25."""
    hw = np.array(hw if hw is not None else [[40, 50]] * B, np.int32)
    f = np.array(f if f is not None else [2.0] * B, np.float64)
    num = np.array(num if num is not None else [2] * B, np.int32)
    wmax = np.array(wmax if wmax is not None else [64] * B, np.int32)
    outs = np.array(outs if outs is not None else [FAKE + (k << 20) for k in range(B)], np.uint64)
    planes = np.array(planes if planes is not None else [FAKE + (k << 24) for k in range(3 * B)], np.uint64)
    nbytes = np.array(nbytes if nbytes is not None else [2000, 500, 500] * B, np.uint64)
    offs = np.array(offs if offs is not None else [0] * (3 * B), np.int64)
    strides = np.array(strides if strides is not None else [[50, 1], [25, 1], [25, 1]] * B, np.int64)
    arrs = (planes, nbytes, offs, strides, hw, f, num, wmax, outs) if descriptors else (None,) * 9
    return N.lib.ctpn_line_crops_yuv420_u8(*(N.ptr(a) for a in arrs[:6]), C.c_void_p(lines), B, rows, Hc,
                                           *(N.ptr(a) for a in arrs[6:]), C.c_void_p(status), None)


COMMON_BAD = [
    (dict(descriptors=False), "null descriptor array"),
    (dict(B=0), "batch = 0, must be 1..64"),
    (dict(B=65), "batch = 65, must be 1..64"),
    (dict(Hc=1), "crop height 1, must be 2..256"),
    (dict(Hc=257), "crop height 257, must be 2..256"),
    (dict(rows=-1, num=[0, 0, 0]), "rows = -1"),
    (dict(num=[2, 11, 2]), "image 1: 11 lines, must be 0..rows = 10"),
    (dict(num=[2, 2, -1]), "image 2: -1 lines"),
    (dict(f=[1.0, 0.0, 1.0]), "image 1: resize factor 0, must be finite and > 0"),
    (dict(f=[-0.5, 1.0, 1.0]), "image 0: resize factor -0.5"),
    (dict(f=[1.0, 1.0, np.nan]), "image 2: resize factor nan"),
    (dict(f=[1.0, np.inf, 1.0]), "image 1: resize factor inf"),
    (dict(outs=[FAKE, 0, FAKE]), "image 1: null output with 2 lines"),
    (dict(wmax=[64, 64, 1]), "image 2: padded width 1, must be 2..1048576"),
    (dict(wmax=[(1 << 20) + 1, 64, 64]), "image 0: padded width 1048577"),
    (dict(lines=0), "null lines or status"),
    (dict(status=0), "null lines or status"),
]

STRIDED_BAD = COMMON_BAD + [
    (dict(srcs=[FAKE, 0, FAKE]), "image 1: null source"),
    (dict(hw=[[40, 50], [0, 50], [40, 50]]), "image 1: bad source size 0 x 50"),
    (dict(nbytes=[6000, 5999, 6000]), "image 1: the box spans bytes [0, 5999]"),
    (dict(offs=[0, 0, 1]), "image 2: the box spans bytes [1, 6000]"),
    (dict(offs=[2, 0, 0], strides=[[150, 3, -1], [150, 3, 1], [150, 3, 1]], nbytes=[5999, 6000, 6000]),
     "image 0: the box spans bytes [0, 5999] of its allocation, outside [0, 5999)"),
    (dict(offs=[5851, 0, 0], strides=[[-150, 3, 1], [150, 3, 1], [150, 3, 1]]), "image 0: the box spans bytes [1, 6000]"),
    (dict(strides=[[150, 3, 1], [150, 1 << 32, 1], [150, 3, 1]]), "image 1: column / channel stride (4294967296, 1)"),
    (dict(strides=[[150, 3, 1], [150, 3, 1], [150, 3, -(1 << 31) - 1]]), "image 2: column / channel stride"),
]

YUV_BAD = COMMON_BAD + [
    (dict(hw=[[40, 50], [41, 50], [40, 50]]), "image 1: source size 41 x 50 must be even and positive"),
    (dict(hw=[[40, 50], [40, 50], [40, 51]]), "image 2: source size 40 x 51 must be even"),
    (dict(planes=[FAKE] * 4 + [0] + [FAKE] * 4), "image 1: null U plane"),
    (dict(nbytes=[2000, 500, 500, 1999, 500, 500, 2000, 500, 500]), "image 1: the Y plane spans bytes [0, 1999]"),
    (dict(nbytes=[2000, 500, 499] + [2000, 500, 500] * 2), "image 0: the V plane spans bytes"),
    (dict(offs=[0] * 7 + [1, 0]), "image 2: the U plane spans bytes [1, 500]"),
    (dict(strides=[[50, 1], [25, 1], [25, 1 << 32]] + [[50, 1], [25, 1], [25, 1]] * 2),
     "image 0: V plane column stride 4294967296 outside the 32-bit range"),
]


@pytest.mark.parametrize("kwargs,match", STRIDED_BAD, ids=[m for _, m in STRIDED_BAD])
def test_strided_crops_refuse_bad_arguments(kwargs, match):
    assert strided_call(**kwargs) == N.ERR_INVALID
    assert match in N.last_error() and "ctpn_line_crops_strided_u8" in N.last_error(), N.last_error()


@pytest.mark.parametrize("kwargs,match", YUV_BAD, ids=[m for _, m in YUV_BAD])
def test_yuv420_crops_refuse_bad_arguments(kwargs, match):
    assert yuv_call(**kwargs) == N.ERR_INVALID
    assert match in N.last_error() and "ctpn_line_crops_yuv420_u8" in N.last_error(), N.last_error()


def test_valid_calls_reach_the_device_check():
    """Valid calls -- negative and zero strides, 64 images, an image without lines and without output -- get as far as the
    device check on a machine without a GPU (so each refusal above came from its own rule)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("the device check is the GPU-less machine's answer; the GPU tests launch real calls")
    assert strided_call() == N.ERR_NO_DEVICE
    assert strided_call(num=[2, 0, 2], outs=[FAKE, 0, FAKE], wmax=[64, 0, 64]) == N.ERR_NO_DEVICE
    rgb_flipped_up = [[-150, 3, -1], [0, 3, 1], [150, 0, 0]]          # bottom-up RGB, one row broadcast, one pixel broadcast
    assert strided_call(strides=rgb_flipped_up, offs=[5852, 0, 0]) == N.ERR_NO_DEVICE
    assert strided_call(B=64) == N.ERR_NO_DEVICE
    assert yuv_call() == N.ERR_NO_DEVICE
    assert yuv_call(B=64, num=[0] * 63 + [2]) == N.ERR_NO_DEVICE
    assert yuv_call(num=[0, 0, 0], lines=0, status=0) == N.ERR_NO_DEVICE


# ---- the engine --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("value", ["canvas", "Source", None, 1, b"source"])
def test_engine_refuses_a_bad_crop_from(value):
    with pytest.raises(ValueError, match="crop_from must be 'resized' or 'source'"):
        check_crop_from(value, 32, "detect_lines_images")


def test_source_crops_need_a_crop_height():
    with pytest.raises(ValueError, match="stream_lines_images: crop_from='source' needs a crop_height"):
        check_crop_from("source", None, "stream_lines_images")
    for crop_from, hc in (("resized", None), ("resized", 32), ("source", 2)):
        check_crop_from(crop_from, hc, "detect_lines_images")


def test_a_stream_with_source_crops_uploads_whole_photos():
    """Source crops stream host photos with compact_rows off: no row maps, every image whole, h * w * 3 bytes each plus the
    28-byte sizes and im_info tail -- 36.6 MB for a 3024 x 4032 photo where the compacted upload sends 14.5 MB."""
    shapes = [(3024, 4032), (4032, 3024), (1080, 1920), (600, 900)]
    items = frontend_plan(shapes)
    assert items[0].rows is not None and items[1].rows is not None
    whole = stream_layout(items, shapes, compact_rows=False)
    assert whole.maps is None and all(r is None for r in whole.rows)
    assert list(whole.stored) == [h for h, w in shapes]
    assert whole.total == (sum(h * w * 3 for h, w in shapes) + 3) // 4 * 4 + 28 * len(shapes)
    compact = stream_layout(items, shapes)
    assert compact.maps is not None and compact.total < whole.total
    assert stream_layout(items[:1], shapes[:1], compact_rows=False).total == 3024 * 4032 * 3 + 28
