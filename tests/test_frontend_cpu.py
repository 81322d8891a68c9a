"""CPU: the device front-end's host side.  frontend_plan (what resize_im and _get_image_blob do to each image) agrees with
the oracle's restatement of resize_im / cvRound and with the repo's own _im_scale, and the two ragged ABI calls
(ctpn_resize_linear_u8_ragged, ctpn_image_blob_f32_ragged) reject every bad descriptor before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

from ctpn_b200 import _native as N
from ctpn_b200.engine import frontend_plan
from oracle import resize as R


def _host_front_end(h, w):
    """(f, resized, im_scale, blob) as ctpn_batch computes them: oracle resize_im / cvRound, then lib's _im_scale."""
    pytest.importorskip("cv2")
    from lib.fast_rcnn.test import _im_scale
    f = R.resize_im_scale(h, w)
    rh, rw = R.out_size(h, w, f, f)
    s = _im_scale((rh, rw, 3))[0]
    blob = (rh, rw) if s == 1.0 else R.out_size(rh, rw, s, s)
    return f, (rh, rw), s, blob


@pytest.mark.parametrize("h,w,what", [(600, 900, "f = 1"), (240, 400, "upscale x2.5"), (37, 53, "upscale, odd"),
                                      (1200, 1800, "exact 1/2"), (65, 63, "upscale of the odd 1/2 kernel case"),
                                      (600, 1100, "5:3 branch: float rescale to MAX_SIZE"), (1000, 3000, "3:1"),
                                      (4032, 3024, "portrait camera photo"), (3024, 4032, "landscape camera photo"),
                                      (1080, 1920, "16:9"), (1920, 1080, "9:16"), (480, 640, "VGA"), (1001, 1667, "just over 5:3")])
def test_plan_matches_the_host_front_end(h, w, what):
    p = frontend_plan([(h, w, 3)])[0]
    f, resized, s, blob = _host_front_end(h, w)
    assert p.f == f and p.resized == resized and p.im_scale == s and p.blob == blob, what
    assert p.dtype == ("|u1" if s == 1.0 else "<f4"), what
    assert frontend_plan([np.zeros((h, w, 3), np.uint8)]) == [p]       # arrays and shape tuples plan alike


def test_plan_cases_take_the_intended_branches():
    one, half, wide, thin = frontend_plan([(600, 900), (1200, 1800), (600, 1100), (1000, 3000)])
    assert one.f == 1.0 and one.dtype == "|u1" and one.blob == (600, 900)
    assert half.f == 0.5 and half.resized == (600, 900) and half.dtype == "|u1"
    assert wide.f == 1.0 and wide.im_scale == 1000.0 / 1100 and wide.dtype == "<f4" and wide.blob == (545, 1000)
    assert thin.f == 1200.0 / 3000 and thin.resized == (400, 1200) and thin.im_scale == 1000.0 / 1200 and thin.blob == (333, 1000)


def test_plan_without_resize_is_the_blob_only():
    pytest.importorskip("cv2")
    from lib.fast_rcnn.test import _im_scale
    for h, w in [(600, 900), (600, 1100), (400, 1200), (37, 53)]:
        p = frontend_plan([(h, w, 3)], resize=False)[0]
        s = _im_scale((h, w, 3))[0]
        assert p.f == 1.0 and p.resized == (h, w) and p.im_scale == s
        assert p.blob == ((h, w) if s == 1.0 else R.out_size(h, w, s, s))


def test_plan_follows_cfg():
    p = frontend_plan([(600, 1100)], cfg={"MAX_SIZE": 1200})[0]
    assert p.im_scale == 1.0 and p.dtype == "|u1"


@pytest.mark.parametrize("image,resize", [
    ((1, 500, 3), True),             # 1-px-thin: resize_im -> 2 x 1200, blob 2 x 1000
    ((1, 5000, 3), True),            # resize_im would make it 0 rows high
    ((3, 1000, 3), True),            # blob 3 x 1000
    ((10, 2000, 3), False),          # already at scale: blob 5 x 1000
])
def test_plan_rejects_degenerate_images(image, resize):
    with pytest.raises(ValueError):
        frontend_plan([image], resize=resize)


def test_plan_takes_small_images_but_only_bgr_uint8():
    assert frontend_plan([(15, 15, 3)], resize=False)[0].blob == (600, 600)
    for bad in (np.zeros((15, 15, 3), np.float32), np.zeros((15, 15), np.uint8), np.zeros((15, 15, 4), np.uint8)):
        with pytest.raises(ValueError):
            frontend_plan([bad])


# ---- the ragged ABI: validation before any CUDA call ------------------------------------------------------------------

def _descriptors(B=3):
    """Valid descriptors of B images packed back to back (image 1 with a row pitch > w), canvas 64 x 96."""
    srcs = [(40, 60, 60, 1.5), (30, 50, 56, 0.5), (64, 96, 96, 1.0)] * ((B + 2) // 3)
    srcs = srcs[:B]
    offs, o = [], 0
    for h, w, pitch, _ in srcs:
        offs.append(o)
        o += h * pitch * 3
    hwp = np.array([[h, w, pitch] for h, w, pitch, _ in srcs], np.int32)
    fxy = np.array([[f, f] for *_, f in srcs], np.float64)
    dst = np.array([R.out_size(h, w, f, f) for h, w, _, f in srcs], np.int32)
    return dict(elems=o, offs=np.array(offs, np.int64), hwp=hwp, fxy=fxy, dst=dst, B=B, H=64, W=96)


_FAKE = C.c_void_p(0x1000)          # never dereferenced: every call below fails validation first


def _call(kind, d, src=_FAKE, dst=_FAKE, lut=_FAKE, offs=True, hwp=True, fxy=True, dhw=True):
    a = (src, d["elems"], N.ptr(d["offs"]) if offs else None, N.ptr(d["hwp"]) if hwp else None,
         N.ptr(d["fxy"]) if fxy else None, N.ptr(d["dst"]) if dhw else None)
    if kind == "u8":
        return N.lib.ctpn_resize_linear_u8_ragged(*a, d["B"], 3, dst, d["H"], d["W"], None)
    return N.lib.ctpn_image_blob_f32_ragged(*a, lut, d["B"], dst, d["H"], d["W"], None)


KINDS = ["u8", "f32"]


@pytest.mark.parametrize("kind", KINDS)
def test_the_baseline_descriptors_are_valid(kind):
    import torch
    if torch.cuda.is_available():
        pytest.skip("the baseline call would launch on the fake pointers; only meaningful without a GPU")
    assert _call(kind, _descriptors()) == N.ERR_NO_DEVICE          # past validation, stopped at the device query


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("B", [0, 65])
def test_batch_size_out_of_range(kind, B):
    d = _descriptors(max(B, 1))
    d["B"] = B
    assert _call(kind, d) == N.ERR_INVALID and "B = %d" % B in N.last_error()


@pytest.mark.parametrize("kind", KINDS)
def test_dst_must_be_the_cvround_size(kind):
    d = _descriptors()
    d["dst"][1, 1] += 1
    assert _call(kind, d) == N.ERR_INVALID and "image 1" in N.last_error() and "cv2 would produce" in N.last_error()


@pytest.mark.parametrize("kind", KINDS)
def test_output_must_fit_the_canvas(kind):
    d = _descriptors()
    d["W"] = 89                                    # image 0: 40 x 60 at 1.5 -> 60 x 90
    assert _call(kind, d) == N.ERR_INVALID and "image 0" in N.last_error() and "canvas" in N.last_error()


@pytest.mark.parametrize("kind", KINDS)
def test_source_extent_within_src_elems(kind):
    d = _descriptors()
    d["elems"] -= 1                                # image 2 ends exactly at the end of the packed sources
    assert _call(kind, d) == N.ERR_INVALID and "image 2" in N.last_error() and "src_elems" in N.last_error()
    d = _descriptors()
    d["offs"][1] = -3
    assert _call(kind, d) == N.ERR_INVALID and "image 1" in N.last_error()
    d = _descriptors()
    d["offs"][0] = (1 << 62)                       # no wrap-around in the extent arithmetic
    assert _call(kind, d) == N.ERR_INVALID and "image 0" in N.last_error()


@pytest.mark.parametrize("kind", KINDS)
def test_pitch_at_least_width(kind):
    d = _descriptors()
    d["hwp"][0, 2] = 59
    assert _call(kind, d) == N.ERR_INVALID and "image 0" in N.last_error() and "pitch" in N.last_error()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("bad", [0.0, -0.5, float("nan")])
def test_scales_must_be_positive(kind, bad):
    for col in (0, 1):
        d = _descriptors()
        d["fxy"][2, col] = bad
        assert _call(kind, d) == N.ERR_INVALID and "image 2" in N.last_error()


@pytest.mark.parametrize("kind", KINDS)
def test_null_pointers(kind):
    d = _descriptors()
    for kw in ({"src": None}, {"dst": None}, {"offs": False}, {"hwp": False}, {"fxy": False}, {"dhw": False}):
        assert _call(kind, d, **kw) == N.ERR_INVALID and "null" in N.last_error(), kw
    if kind == "f32":
        assert _call(kind, d, lut=None) == N.ERR_INVALID and "null" in N.last_error()


def test_bad_channel_count():
    d = _descriptors()
    for ch in (0, 5):
        assert N.lib.ctpn_resize_linear_u8_ragged(_FAKE, d["elems"], N.ptr(d["offs"]), N.ptr(d["hwp"]), N.ptr(d["fxy"]),
                                                  N.ptr(d["dst"]), d["B"], ch, _FAKE, d["H"], d["W"], None) == N.ERR_INVALID
