"""GPU: the ragged device front-end.  ctpn_resize_linear_u8_ragged / ctpn_image_blob_f32_ragged write every image of a
mixed batch bit-identically to the single-image kernels, to the oracle's restatement of OpenCV and (uint8) to cv2.resize,
and leave the canvas padding untouched; Engine.detect_images / rois_images equal the per-image device path in every
arithmetic, and the host front-end of test_ctpn; ctpn/demo.py --device-frontend writes the files --batch writes."""
import contextlib

import numpy as np
import pytest
import torch

from oracle import resize as R, synth

pytestmark = pytest.mark.gpu

MEANS = np.array([[[102.9801, 115.9465, 122.7717]]])
# (h, w, f of the uint8 resize, scale of the float blob): odd borders, upscales, exact 1/2 (INTER_AREA routing, also with
# odd sides), f = 1, a 3:1 image, both orientations
KERNEL_CASES = [(37, 53, 1.5, 0.73), (1200, 1800, 0.5, 1000.0 / 1800), (65, 63, 0.5, 0.5), (600, 900, 1.0, 1.0),
                (1000, 3000, 0.4, 1000.0 / 3000), (480, 640, 1.25, 1.5), (301, 203, 0.5, 0.5), (90, 160, 600 / 90.0, 2.0),
                (756, 1008, 600 / 756.0, 1000.0 / 1008), (1008, 756, 600 / 756.0, 0.6), (300, 560, 1.0, 1000.0 / 560),
                (17, 400, 3.0, 0.5)]
PITCH_PAD = [0, 3, 17, 0, 5, 0, 1, 64, 0, 2, 0, 9]          # row pitch = w + pad (pixels)


@pytest.fixture(scope="module")
def weights():
    return synth.make_weights(0)


@contextlib.contextmanager
def ipp_off():
    import cv2
    prev = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        yield cv2
    finally:
        cv2.ipp.setUseIPP(prev)


def pack(images, pads, seed=0):
    """Sources packed back to back with row pitch w + pad and a gap after each image, garbage in pitch and gaps."""
    rs = np.random.RandomState(seed)
    offs, hwp, parts, o = [], [], [], 0
    for im, pad in zip(images, pads):
        h, w = im.shape[:2]
        block = rs.randint(0, 256, (h, w + pad, 3)).astype(np.uint8)
        block[:, :w] = im
        gap = rs.randint(0, 256, 7 * 3).astype(np.uint8)
        parts += [block.ravel(), gap]
        offs.append(o)
        hwp.append((h, w, w + pad))
        o += block.size + gap.size
    return np.concatenate(parts), np.array(offs, np.int64), np.array(hwp, np.int32)


def test_ragged_kernels_equal_single_image_kernels_oracle_and_cv2():
    from ctpn_b200 import Engine, _native as N
    eng = Engine(None)
    images = [synth.make_image(200 + i, h, w) for i, (h, w, _, _) in enumerate(KERNEL_CASES)]
    flat, offs, hwp = pack(images, PITCH_PAD)
    src = torch.from_numpy(flat).cuda()
    B = len(images)
    for kind in ("u8", "f32"):
        col = 2 if kind == "u8" else 3
        fxy = np.array([[c[col], c[col]] for c in KERNEL_CASES], np.float64)
        dst_hw = np.array([R.out_size(c[0], c[1], c[col], c[col]) for c in KERNEL_CASES], np.int32)
        H, W = int(dst_hw[:, 0].max()) + 3, int(dst_hw[:, 1].max()) + 5
        if kind == "u8":
            canvas = torch.full((B, H, W, 3), 0xA5, dtype=torch.uint8, device="cuda")
            rc = N.lib.ctpn_resize_linear_u8_ragged(N.ptr(src), flat.size, N.ptr(offs), N.ptr(hwp), N.ptr(fxy), N.ptr(dst_hw), B, 3,
                                                    N.ptr(canvas), H, W, N.stream_ptr())
        else:
            canvas = torch.full((B, H, W, 3), -12345.5, dtype=torch.float32, device="cuda")
            rc = N.lib.ctpn_image_blob_f32_ragged(N.ptr(src), flat.size, N.ptr(offs), N.ptr(hwp), N.ptr(fxy), N.ptr(dst_hw),
                                                  N.ptr(eng._mean_lut()), B, N.ptr(canvas), H, W, N.stream_ptr())
        N.check(rc, "ragged " + kind)
        got = canvas.cpu().numpy()
        for b, (im, (dh, dw)) in enumerate(zip(images, dst_hw)):
            f = float(fxy[b, 0])
            what = "%s image %d (%dx%d at %r)" % (kind, b, im.shape[0], im.shape[1], f)
            if kind == "u8":
                single = eng.resize_images(im[None], f)[0].cpu().numpy()
                np.testing.assert_array_equal(got[b, :dh, :dw], single, what)
                np.testing.assert_array_equal(single, R.resize_linear_u8(im, f), what)
                import cv2
                np.testing.assert_array_equal(single, cv2.resize(im, None, None, fx=f, fy=f, interpolation=cv2.INTER_LINEAR), what)
                pad = 0xA5
            else:
                single = eng.image_blob(im[None], f)[0].cpu().numpy()
                assert np.array_equal(got[b, :dh, :dw].view(np.uint32), single.view(np.uint32)), what
                ref = im.astype(np.float32)
                ref -= MEANS
                assert np.array_equal(single.view(np.uint32), R.resize_linear_f32(ref, f).view(np.uint32)), what
                pad = np.float32(-12345.5)
            assert (got[b, dh:] == pad).all() and (got[b, :dh, dw:] == pad).all(), what + ": padding was written"


# raw photo sizes -> every branch of the front-end: upscale to (600, 1000) u8; exact 1/2 u8; 5:3+ -> float rescale;
# 3:1 -> float rescale; portrait u8; odd tiny upscale; f = 1
PHOTOS = [(240, 400), (1200, 1800), (300, 550), (200, 600), (450, 300), (37, 53), (600, 900)]


def make_photos(seed0=300):
    return [synth.make_image(seed0 + i, h, w) for i, (h, w) in enumerate(PHOTOS)]


def single_image_rois(eng, im, p):
    """The per-image device path: Engine.resize_images, then image_blob (or the uint8 image itself), then the detector."""
    resized = eng.resize_images(im[None], p.f)
    blob = resized if p.dtype == "|u1" else eng.image_blob(resized, p.im_scale)
    assert tuple(blob.shape[1:3]) == p.blob
    return eng.rois_batch(blob, np.array([[p.blob[0], p.blob[1], p.im_scale]], np.float32))[0]


@pytest.mark.parametrize("mode", ["bf16x2", "f16f8", "bf16x3p"])
def test_detect_images_equals_single_image_runs(weights, mode):
    from ctpn_b200 import Engine, frontend_plan
    eng = Engine(weights, mode=mode)
    photos = make_photos()
    plan = frontend_plan(photos)
    assert {p.dtype for p in plan} == {"|u1", "<f4"}
    got = eng.rois_images(photos, max_batch=3)          # f16f8: the first ragged batch calibrates the scales
    det = eng.detect_images(photos, max_batch=3)
    for i, (im, p) in enumerate(zip(photos, plan)):
        rois, im_scale, f = got[i]
        assert im_scale == p.im_scale and f == p.f
        want = single_image_rois(eng, im, p)
        assert rois.shape[0] > 0 and np.array_equal(rois, want), "%s image %d %s" % (mode, i, im.shape)
        scores, boxes, f2 = det[i]
        assert f2 == p.f and boxes.dtype == np.float64
        assert np.array_equal(scores, want[:, 0]) and np.array_equal(boxes, want[:, 1:5] / np.float64(p.im_scale))


def test_detect_images_equals_test_ctpn_on_the_host_resize(weights):
    """cv2's resize_im + test_ctpn (its _get_image_blob on the host) == detect_images, with OpenCV's own float code."""
    from ctpn import demo
    from ctpn_b200 import Session
    from lib.fast_rcnn.test import test_ctpn
    from lib.networks.factory import get_network
    sess = Session(weights, planes=2)
    net = get_network("VGGnet_test")
    photos = make_photos(seed0=400)
    with ipp_off():
        got = sess.engine.detect_images(photos, max_batch=4, return_resized=True)
        for i, im in enumerate(photos):
            img, f = demo.resize_im(im, scale=600, max_scale=1200)
            scores, boxes = test_ctpn(sess, net, img)
            s2, b2, f2, resized = got[i]
            assert f2 == f and np.array_equal(resized, img), i
            assert np.array_equal(s2, scores) and np.array_equal(b2, boxes) and b2.dtype == boxes.dtype, i


def test_resize_false_runs_the_blob_only(weights):
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="bf16x2")
    photos = make_photos(seed0=500)
    full = eng.detect_images(photos, return_resized=True)
    resized = [r[3] for r in full]
    again = eng.detect_images(resized, resize=False)
    for (s0, b0, _, _), (s1, b1, f1) in zip(full, again):
        assert f1 == 1.0 and np.array_equal(s0, s1) and np.array_equal(b0, b1)
    with pytest.raises(ValueError):
        eng.detect_images([photos[0].astype(np.float32)])
    with pytest.raises(ValueError):
        eng.detect_images([np.zeros((1, 500, 3), np.uint8)])
    with pytest.raises(ValueError):
        eng.detect_images(photos, max_batch=65)


def test_demo_device_frontend_writes_the_same_files(weights, tmp_path, monkeypatch):
    """ctpn/demo.py --batch 4 --device-frontend == --batch 4 (IPP off): res_*.txt and the annotated images, byte for byte.
    Among the images: one wider than 5:3 (float rescale of the blob) and one at exactly 1/2 (INTER_AREA routing)."""
    from ctpn import demo
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **weights)
    folder = tmp_path / "images"
    folder.mkdir()
    with ipp_off() as cv2:
        for i, (h, w) in enumerate([(300, 560), (1200, 1600), (480, 360), (200, 500), (240, 240), (350, 420)]):
            cv2.imwrite(str(folder / ("im_%d.png" % i)), synth.make_image(70 + i, h, w))
        out = {}
        for flags in ([], ["--device-frontend"]):
            res = tmp_path / ("results_%d" % len(flags))
            monkeypatch.setattr(demo, "RESULTS_DIR", str(res))
            demo.main(["--weights", npz, "--planes", "2", "--images", str(folder / "*.png"), "--batch", "4"] + flags)
            out[len(flags)] = {p.name: p.read_bytes() for p in sorted(res.iterdir())}
    assert len(out[0]) == 12 and sorted(out[0]) == sorted(out[1])
    for name in out[0]:
        assert out[0][name] == out[1][name], name
