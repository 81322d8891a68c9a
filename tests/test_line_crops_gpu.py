"""GPU: text-line crops on the device.  ctpn_line_crops_u8 equals oracle/crop.py bit for bit, writes zeros past each line's
width and nothing outside each image's [m, Hc, Wmax, 3]; detect_lines_images(crop_height=32) returns crops equal to
cv2.warpAffine on its own resize_im output for host arrays, BGR / RGB tensors and crop views, NV12 and I420 frames,
float32-blob batches, resize=False and modes H and O; stream_lines_images equals the list call; the crops outlive a
stream closed early; and (tests/line_crops_cases.py, in a process of its own) they add no copy and no synchronise."""
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

from device_image_checks import BGR_LAYOUTS, RGB_LAYOUTS, device_list, photos
from oracle import crop
from yuv_frames import device_frame, video_photos

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SENTINEL = 0xA5
# connector score thresholds low enough that the synthetic weights give the photos lines to cut; chains of at least two
# proposals of the default width, as with the default thresholds
LOW = (0.05, 0.2, 50, 0.5, 0.5, 0.0, 0.0, 16, 2)


@pytest.fixture(scope="module")
def engine():
    from ctpn_b200 import Engine
    from oracle import synth
    return Engine(synth.make_weights(0), mode="bf16x2")


@pytest.fixture(scope="module")
def images():
    """The mixed photos (upscales, exact 1/2, a 3:1 image whose blob is a float32 rescale, portrait, tiny, f = 1) and a
    flat one."""
    return photos(16) + [np.full((300, 420, 3), 128, np.uint8)]


def cv2_crop(im, line, Hc):
    Wc = crop.crop_width(line, Hc)
    return cv2.warpAffine(im, crop.crop_matrix(line, Hc, Wc), (Wc, Hc), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP,
                          borderMode=cv2.BORDER_REPLICATE)


# ---- the kernel against the oracle -----------------------------------------------------------------------------------------

def random_lines(rng, m, h, w):
    out = np.empty((m, 9))
    for j in range(m):
        x1, y1 = rng.uniform(-0.2 * w, 1.1 * w), rng.uniform(-0.2 * h, 1.1 * h)
        if j % 3 == 0:
            x1, y1 = np.round(x1), np.floor(y1) + 0.5
        a, L, H = rng.uniform(-0.5, 0.5), rng.uniform(1, w), (0.0 if j % 7 == 3 else rng.uniform(1, 0.5 * h))
        x2, y2, x3, y3 = x1 + L * np.cos(a), y1 + L * np.sin(a), x1 - H * np.sin(a), y1 + H * np.cos(a)
        out[j] = [x1, y1, x2, y2, x3, y3, x2 + x3 - x1, y2 + y3 - y1, 0.9]
    return out


def run_kernel(canvas, hw, lines_dev, num, wmax, Hc, gap=4096):
    """ctpn_line_crops_u8 into views of one sentinel-filled buffer, with gaps between the images' outputs.  Returns
    (the whole buffer, per image (offset, shape)), status."""
    from ctpn_b200 import _native as N
    B, rows = lines_dev.shape[:2]
    shapes = [(int(m), Hc, int(w), 3) for m, w in zip(num, wmax)]
    offs = np.cumsum([gap] + [int(np.prod(s)) + gap for s in shapes[:-1]])
    buf = torch.full((int(offs[-1] + np.prod(shapes[-1]) + gap),), SENTINEL, dtype=torch.uint8, device="cuda")
    ptrs = np.array([buf.data_ptr() + int(o) for o in offs], np.uint64)
    status = torch.zeros(B, dtype=torch.int32, device="cuda")
    Hr, Wr = canvas.shape[1:3]
    hw, num, wmax = (np.ascontiguousarray(v, np.int32) for v in (hw, num, wmax))      # alive across the call
    N.check(N.lib.ctpn_line_crops_u8(N.ptr(canvas), Hr * Wr * 3, Wr * 3, N.ptr(hw), N.ptr(lines_dev), B, rows, Hc, N.ptr(num),
                                     N.ptr(wmax), N.ptr(ptrs), N.ptr(status), N.stream_ptr()), "ctpn_line_crops_u8")
    return buf.cpu().numpy(), list(zip(offs, shapes)), status.cpu().numpy()


@pytest.mark.parametrize("Hc", [2, 32, 256])
def test_kernel_equals_the_oracle(Hc):
    rng = np.random.default_rng(Hc)
    hw = np.array([[60, 90], [17, 300], [200, 40], [33, 33], [120, 160]], np.int32)
    num = [5, 0, 7, 1, 12]
    B, rows, (Hr, Wr) = len(hw), 14, (hw[:, 0].max() + 3, hw[:, 1].max() + 5)
    canvas = rng.integers(0, 256, (B, Hr, Wr, 3), dtype=np.uint8)       # the padding holds bytes a stray read would see
    lines = rng.uniform(-1e3, 1e3, (B, rows, 9))                        # rows past num[b] are never read
    want, wmax = [], []
    for b, (h, w) in enumerate(hw):
        lines[b, :num[b]] = random_lines(rng, num[b], h, w)
        crops, widths = crop.line_crops(canvas[b, :h, :w], lines[b, :num[b]], Hc)
        want.append(crops)
        wmax.append(int(widths.max()) if num[b] else 0)
    buf, where, status = run_kernel(torch.from_numpy(canvas).cuda(), hw, torch.from_numpy(lines).cuda(), num, wmax, Hc)
    assert not status.any()
    seen = np.zeros(buf.size, bool)
    for b, (o, shape) in enumerate(where):
        n = int(np.prod(shape))
        assert np.array_equal(buf[o:o + n].reshape(shape), want[b]), b          # zeros past each width included
        seen[o:o + n] = True
    assert (buf[~seen] == SENTINEL).all()


def test_a_width_the_kernel_disagrees_with_gets_no_pixels():
    """A padded width below a line's Wc, or a line with no finite width, sets the image's status and leaves that line's
    output unwritten; the image's other lines and the other images are cut as usual.  Lines far outside the canvas read
    clamped taps only."""
    rng = np.random.default_rng(3)
    hw = np.array([[50, 70], [50, 70]], np.int32)
    canvas = rng.integers(0, 256, (2, 50, 70, 3), dtype=np.uint8)
    lines = np.stack([random_lines(rng, 4, 50, 70), random_lines(rng, 4, 50, 70)])
    lines[1, 1, :6] = [1e15, -1e15, 1e15 + 4096, -1e15, 1e15, -1e15 + 4096]  # finite, far outside: taps clamp to a corner
    lines[1, 2, 0] = np.nan
    widths = [crop.crop_widths(lines[0], 32), crop.crop_widths(np.delete(lines[1], 2, 0), 32)]
    wmax = [int(widths[0].max()) - 1, int(widths[1].max())]    # the widest line of image 0 no longer fits
    buf, where, status = run_kernel(torch.from_numpy(canvas).cuda(), hw, torch.from_numpy(lines).cuda(), [4, 4], wmax, 32)
    assert list(status) == [1, 1]
    for b in range(2):
        o, shape = where[b]
        out = buf[o:o + int(np.prod(shape))].reshape(shape)
        for j in range(4):
            if b == 1 and j == 2:
                assert (out[j] == SENTINEL).all()
                continue
            wc = crop.crop_width(lines[b, j], 32)
            if wc > wmax[b]:
                assert (out[j] == SENTINEL).all(), (b, j)
            elif not (b == 1 and j == 1):
                assert np.array_equal(out[j, :, :wc], crop.line_crop(canvas[b], lines[b, j], 32)), (b, j)
                assert (out[j, :, wc:] == 0).all()


# ---- the engine ---------------------------------------------------------------------------------------------------------

def check_crops(results, Hc=32, plain=None):
    """Every result (lines, f, crops, widths, resized): crops equal cv2.warpAffine on resized, zeros past the widths; and
    (lines, f) equal the crop_height=None call's `plain` results."""
    total = 0
    for i, r in enumerate(results):
        lines, f, crops, widths, resized = r
        if plain is not None:
            assert len(plain[i]) == 3 and np.array_equal(plain[i][0], lines) and plain[i][1] == f
            assert np.array_equal(plain[i][2], resized)
        m = len(lines)
        assert crops.is_cuda and crops.dtype == torch.uint8 and widths.dtype == np.int64
        assert np.array_equal(widths, crop.crop_widths(lines, Hc))
        assert tuple(crops.shape) == (m, Hc, int(widths.max()) if m else 0, 3)
        c = crops.cpu().numpy()
        for j in range(m):
            assert np.array_equal(c[j, :, :widths[j]], cv2_crop(resized, lines[j], Hc)), (i, j)
            assert (c[j, :, widths[j]:] == 0).all()
        total += m
    return total


@pytest.mark.parametrize("mode", ["H", "O"])
def test_list_call_on_host_arrays(engine, images, mode):
    from ctpn_b200 import frontend_plan
    assert {p.dtype for p in frontend_plan(images)} == {"|u1", "<f4"}           # uint8 and float32-blob batches
    plain = engine.detect_lines_images(images, cfg=LOW, mode=mode, return_resized=True)
    got = engine.detect_lines_images(images, cfg=LOW, mode=mode, return_resized=True, crop_height=32)
    assert check_crops(got, plain=plain) > 0
    small = engine.detect_lines_images(images[:5], cfg=LOW, mode=mode, max_batch=2, crop_height=48)
    assert all(len(r) == 4 for r in small)
    for r, p in zip(small, plain[:5]):
        assert np.array_equal(r[0], p[0])
        for j in range(len(r[0])):
            assert np.array_equal(r[2][j, :, :r[3][j]].cpu().numpy(), cv2_crop(p[2], r[0][j], 48))


def test_batches_without_lines(engine, images):
    """No line passes a minimum score above 1: every image gets an empty [0, Hc, 0, 3] tensor and no kernel runs."""
    cfg = [1.1, 0.2, 50, 0.7, 0.7, 0.5, 0.9, 16, 2]
    for r in engine.detect_lines_images(images[:5], cfg=cfg, crop_height=32):
        assert len(r[0]) == 0 and tuple(r[2].shape) == (0, 32, 0, 3) and r[3].shape == (0,)
    for r in engine.stream_lines_images(iter(images[:5]), cfg=cfg, crop_height=32, max_batch=2):
        assert len(r[0]) == 0 and tuple(r[2].shape) == (0, 32, 0, 3) and r[3].shape == (0,)


def test_list_call_without_resize(engine, images):
    ims = [im for im in images if min(im.shape[:2]) >= 200][:6]
    plain = engine.detect_lines_images(ims, cfg=LOW, resize=False, return_resized=True)
    got = engine.detect_lines_images(ims, cfg=LOW, resize=False, return_resized=True, crop_height=32)
    assert check_crops(got, plain=plain) > 0
    assert all(np.array_equal(p[2], im) for p, im in zip(plain, ims))


@pytest.mark.parametrize("layouts", [BGR_LAYOUTS, RGB_LAYOUTS], ids=["bgr", "rgb"])
def test_list_call_on_tensors(engine, images, layouts):
    tensors, channels = device_list(images, layouts)
    plain = engine.detect_lines_images(images, cfg=LOW, mode="O", return_resized=True)
    got = engine.detect_lines_images(tensors, cfg=LOW, mode="O", return_resized=True, crop_height=32, channels=channels, max_batch=7)
    assert check_crops(got, plain=plain) > 0


@pytest.mark.parametrize("layout", ["NV12", "I420"])
def test_list_call_on_frames(engine, layout):
    ph = video_photos(6)
    frames = [device_frame(*p, layout, seed=i) for i, (_, p) in enumerate(ph)]
    plain = engine.detect_lines_images([b for b, _ in ph], cfg=LOW, return_resized=True)
    got = engine.detect_lines_images(frames, cfg=LOW, return_resized=True, crop_height=32)
    assert check_crops(got, plain=plain) > 0


def same_crop_results(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert len(x) == len(y) == 5, i
        assert np.array_equal(x[0], y[0]) and x[1] == y[1] and np.array_equal(x[3], y[3]) and np.array_equal(x[4], y[4]), i
        assert torch.equal(x[2], y[2]), i


@pytest.mark.parametrize("window,max_batch", [(3, 2), (40, 32)])
def test_stream_equals_the_list_call(engine, images, window, max_batch):
    want = engine.detect_lines_images(images, cfg=LOW, mode="O", return_resized=True, crop_height=32)
    got = list(engine.stream_lines_images(iter(images), cfg=LOW, mode="O", return_resized=True, crop_height=32, window=window,
                                          max_batch=max_batch))
    same_crop_results(got, want)
    tensors, channels = device_list(images, BGR_LAYOUTS)
    got = list(engine.stream_lines_images(iter(tensors), cfg=LOW, mode="O", return_resized=True, crop_height=32, window=window,
                                          max_batch=max_batch))
    same_crop_results(got, want)


def test_crops_outlive_a_stream_closed_early(engine, images):
    want = engine.detect_lines_images(images, cfg=LOW, return_resized=True, crop_height=32)
    gen = engine.stream_lines_images(iter(images), cfg=LOW, return_resized=True, crop_height=32, window=4, max_batch=2)
    kept = [next(gen) for _ in range(5)]
    gen.close()
    junk = [torch.full((1 << 22,), 0x3C, dtype=torch.uint8, device="cuda") for _ in range(8)]   # reuse freed blocks
    del junk
    same_crop_results(engine.detect_lines_images(images, cfg=LOW, return_resized=True, crop_height=32), want)
    same_crop_results(kept, want[:5])
    same_crop_results(list(engine.stream_lines_images(iter(images), cfg=LOW, return_resized=True, crop_height=32)), want)


def test_crops_on_a_side_stream(engine, images):
    """Crops are ready, in stream order, on the stream that was current for the call -- a side stream here."""
    want = engine.detect_lines_images(images[:6], cfg=LOW, return_resized=True, crop_height=32)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        got = engine.detect_lines_images(images[:6], cfg=LOW, return_resized=True, crop_height=32)
        got_s = list(engine.stream_lines_images(iter(images[:6]), cfg=LOW, return_resized=True, crop_height=32, max_batch=2, window=3))
        copies = [r[2].clone() for r in got + got_s]           # on the side stream, after the crop kernels
    side.synchronize()
    for r, w, c in zip(got + got_s, want + want, copies):
        assert torch.equal(c, w[2])



def test_transfer_census():
    """The torch.profiler census of tests/line_crops_cases.py, in a process of its own: profiler sessions are kept out of
    the process that runs the other GPU tests, as tests/test_yuv_frames_gpu.py keeps its census."""
    cmd = [sys.executable, "-m", "pytest", "-q", "-s", "-p", "no:cacheprovider", "-m", "gpu",
           os.path.join(HERE, "line_crops_cases.py") + "::test_transfer_census"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=os.path.dirname(HERE))
    assert p.returncode == 0 and " passed" in p.stdout and "failed" not in p.stdout, \
        "stdout:\n%s\nstderr:\n%s" % (p.stdout[-4000:], p.stderr[-2000:])
