"""GPU: line crops out of the source images (crop_from="source").  ctpn_line_crops_strided_u8 and ctpn_line_crops_yuv420_u8
equal oracle/crop.py on the source lines lines / f bit for bit, write zeros past each width and nothing outside each
image's [m, Hc, Wmax, 3]; detect_lines_images(crop_from="source") equals cv2.warpAffine of the source photo for host
arrays, BGR / RGB tensors and crop views, NV12 and I420 frames, float32-blob batches and modes H and O; with f = 1 source
crops are canvas crops; the stream equals the list call over many batches (its three source buffers) for every input kind
and its crops outlive an early close; and (tests/source_crops_cases.py, in a process of its own) the census of copies,
synchronises and crop launches."""
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

from device_image_checks import BGR_LAYOUTS, RGB_LAYOUTS, device_list, photos
from oracle import crop, yuv
from yuv_frames import device_frame, video_photos

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SENTINEL = 0xA5
# as in tests/test_line_crops_gpu.py: connector thresholds low enough that the synthetic weights give the photos lines
LOW = (0.05, 0.2, 50, 0.5, 0.5, 0.0, 0.0, 16, 2)


@pytest.fixture(scope="module")
def engine():
    from ctpn_b200 import Engine
    from oracle import synth
    return Engine(synth.make_weights(0), mode="bf16x2")


@pytest.fixture(scope="module")
def images():
    return photos(16)


def source_lines(lines, f):
    src = np.array(lines, np.float64).reshape(-1, 9)
    src[:, :8] /= np.float64(f)
    return src


def cv2_source_crop(src_bgr, line, f, Hc):
    ln = source_lines(line, f)[0]
    Wc = crop.crop_width(ln, Hc)
    return cv2.warpAffine(src_bgr, crop.crop_matrix(ln, Hc, Wc), (Wc, Hc), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP,
                          borderMode=cv2.BORDER_REPLICATE)


# ---- the kernels against the oracle --------------------------------------------------------------------------------------

def random_lines(rng, m, rh, rw):
    """m lines of a rh x rw resize_im frame, some partly outside it, some of height 0, some on half pixels."""
    out = np.empty((m, 9))
    for j in range(m):
        x1, y1 = rng.uniform(-0.2 * rw, 1.1 * rw), rng.uniform(-0.2 * rh, 1.1 * rh)
        if j % 3 == 0:
            x1, y1 = np.round(x1), np.floor(y1) + 0.5
        a, L, H = rng.uniform(-0.5, 0.5), rng.uniform(1, rw), (0.0 if j % 7 == 3 else rng.uniform(1, 0.3 * rh))
        x2, y2, x3, y3 = x1 + L * np.cos(a), y1 + L * np.sin(a), x1 - H * np.sin(a), y1 + H * np.cos(a)
        out[j] = [x1, y1, x2, y2, x3, y3, x2 + x3 - x1, y2 + y3 - y1, 0.9]
    return out


def run_kernel(name, desc, src_hw, f, lines, num, Hc, gap=4096):
    """ctpn_line_crops_{strided,yuv420}_u8 of the source descriptors into views of one sentinel-filled buffer with gaps
    between the images' outputs; widths from ctpn_line_crop_widths_host on lines / f.  Returns (the buffer, per image
    (offset, shape), the oracle-free widths), status."""
    from ctpn_b200 import _native as N
    from ctpn_b200.engine import descriptor_arrays
    B, rows = lines.shape[:2]
    wmax = [int(crop.crop_widths(source_lines(lines[b, :num[b]], f[b]), Hc).max()) if num[b] else 0 for b in range(B)]
    shapes = [(int(m), Hc, int(w), 3) for m, w in zip(num, wmax)]
    offs = np.cumsum([gap] + [int(np.prod(s)) + gap for s in shapes[:-1]])
    buf = torch.full((int(offs[-1] + np.prod(shapes[-1]) + gap),), SENTINEL, dtype=torch.uint8, device="cuda")
    ptrs = np.array([buf.data_ptr() + int(o) for o in offs], np.uint64)
    status = torch.zeros(B, dtype=torch.int32, device="cuda")
    addr, nbytes, doffs, strides = descriptor_arrays(desc)
    hw, f64 = np.ascontiguousarray(src_hw, np.int32), np.ascontiguousarray(f, np.float64)
    num32, wmax32 = np.ascontiguousarray(num, np.int32), np.ascontiguousarray(wmax, np.int32)
    lines_dev = torch.from_numpy(np.ascontiguousarray(lines)).cuda()
    N.check(getattr(N.lib, name)(N.ptr(addr), N.ptr(nbytes), N.ptr(doffs), N.ptr(strides), N.ptr(hw), N.ptr(f64),
                                 N.ptr(lines_dev), B, rows, Hc, N.ptr(num32), N.ptr(wmax32), N.ptr(ptrs), N.ptr(status),
                                 N.stream_ptr()), name)
    return buf.cpu().numpy(), list(zip(offs, shapes)), status.cpu().numpy()


def check_against_oracle(buf, where, status, sources_bgr, lines, num, f, Hc):
    assert not status.any()
    seen = np.zeros(buf.size, bool)
    for b, (o, shape) in enumerate(where):
        n = int(np.prod(shape))
        want, _ = crop.line_crops(sources_bgr[b], source_lines(lines[b, :num[b]], f[b]), Hc)
        assert np.array_equal(buf[o:o + n].reshape(shape), want.reshape(shape)), b     # zeros past each width included
        seen[o:o + n] = True
    assert (buf[~seen] == SENTINEL).all()


def strided_sources(rng):
    """(tensor, channels, BGR host copy) in every strided layout: pitched rows (> 3w), RGB through a negative channel
    stride, a crop view, planar CHW, a zero row stride and a zero column stride (broadcasts)."""
    from ctpn_b200.engine import tensor_descriptor  # noqa: F401  (the engine's descriptor builder is what is tested)
    out = []
    im = rng.integers(0, 256, (90, 130, 3), dtype=np.uint8)
    big = torch.from_numpy(rng.integers(0, 256, (90, 160, 3), dtype=np.uint8)).cuda()
    big[:, :130] = torch.from_numpy(im).cuda()
    out.append((big[:, :130], "BGR", im))                                              # row pitch 480 > 390
    rgb = rng.integers(0, 256, (150, 80, 3), dtype=np.uint8)
    out.append((torch.from_numpy(rgb).cuda(), "RGB", np.ascontiguousarray(rgb[:, :, ::-1])))
    frame = torch.from_numpy(rng.integers(0, 256, (300, 400, 3), dtype=np.uint8)).cuda()
    out.append((frame[37:237, 51:351], "BGR", frame[37:237, 51:351].cpu().numpy()))      # crop view
    chw = torch.from_numpy(rng.integers(0, 256, (3, 64, 96), dtype=np.uint8)).cuda()
    out.append((chw.permute(1, 2, 0), "BGR", chw.permute(1, 2, 0).cpu().numpy()))
    row = torch.from_numpy(rng.integers(0, 256, (1, 120, 3), dtype=np.uint8)).cuda()
    out.append((row.expand(70, 120, 3), "BGR", np.broadcast_to(row.cpu().numpy(), (70, 120, 3)).copy()))
    px = torch.from_numpy(rng.integers(0, 256, (60, 1, 3), dtype=np.uint8)).cuda()
    out.append((px.expand(60, 90, 3), "BGR", np.broadcast_to(px.cpu().numpy(), (60, 90, 3)).copy()))
    return out


@pytest.mark.parametrize("Hc", [2, 32, 256])
def test_strided_kernel_equals_the_oracle(Hc):
    from ctpn_b200.engine import tensor_descriptor
    rng = np.random.default_rng(100 + Hc)
    src = strided_sources(rng)
    B, rows = len(src), 12
    f = [rng.uniform(0.3, 4.0) for _ in range(B)]
    f[2] = 1.0
    num = [5, 12, 0, 7, 3, 9]
    lines = rng.uniform(-1e3, 1e3, (B, rows, 9))             # rows past num[b] are never read
    for b, (t, _, bgr) in enumerate(src):
        h, w = bgr.shape[:2]
        lines[b, :num[b]] = random_lines(rng, num[b], h * f[b], w * f[b])
    desc = [tensor_descriptor(t, ch) for t, ch, _ in src]
    buf, where, status = run_kernel("ctpn_line_crops_strided_u8", desc, [b.shape[:2] for _, _, b in src], f, lines, num, Hc)
    check_against_oracle(buf, where, status, [b for _, _, b in src], lines, num, f, Hc)


@pytest.mark.parametrize("Hc", [32, 48])
def test_yuv420_kernel_equals_the_oracle(Hc):
    """All four single-buffer layouts, pitched and split-chroma surfaces, a crop, and a 1920 x 1080 NV12 frame in a
    2048-byte-pitch, 1088-row surface."""
    from ctpn_b200.engine import yuv420_descriptor
    from yuv_frames import random_planes
    rng = np.random.default_rng(200 + Hc)
    layouts = ["NV12", "NV21", "I420", "YV12", "nv12_pitched", "i420_pitched", "nv12_split", "crop", "nv12_padded_surface"]
    sizes = [(64, 96), (120, 90), (38, 54), (200, 300), (100, 140), (48, 64), (80, 80), (60, 100), (1080, 1920)]
    frames, bgr = [], []
    for i, (layout, (h, w)) in enumerate(zip(layouts, sizes)):
        Y, U, V = random_planes(300 + i, h, w)
        frames.append(device_frame(Y, U, V, layout, seed=i))
        bgr.append(cv2.cvtColor(yuv.planes_to_buffer(Y, U, V, "I420"), cv2.COLOR_YUV2BGR_I420))
    assert tuple(frames[-1].y.stride()) == (2048, 1) and frames[-1].u.data_ptr() - frames[-1].y.data_ptr() == 1088 * 2048
    B, rows = len(frames), 10
    f = [rng.uniform(0.3, 3.0) for _ in range(B)]
    f[-1] = 600.0 / 1080
    num = [4, 10, 2, 0, 6, 3, 1, 5, 10]
    lines = rng.uniform(-1e3, 1e3, (B, rows, 9))
    for b, (h, w) in enumerate(sizes):
        lines[b, :num[b]] = random_lines(rng, num[b], h * f[b], w * f[b])
    desc = [d for fr in frames for d in yuv420_descriptor(fr)]
    buf, where, status = run_kernel("ctpn_line_crops_yuv420_u8", desc, sizes, f, lines, num, Hc)
    check_against_oracle(buf, where, status, bgr, lines, num, f, Hc)


def test_yuv420_batches_over_32_frames_launch_in_chunks():
    from ctpn_b200.engine import yuv420_descriptor
    from yuv_frames import random_planes
    rng = np.random.default_rng(7)
    B, rows, Hc = 45, 4, 32
    sizes = [(40 + 2 * (b % 5), 60 + 4 * (b % 3)) for b in range(B)]
    frames, bgr = [], []
    for b, (h, w) in enumerate(sizes):
        Y, U, V = random_planes(500 + b, h, w)
        frames.append(device_frame(Y, U, V, ("NV12", "I420", "YV12", "NV21")[b % 4], seed=b))
        bgr.append(cv2.cvtColor(yuv.planes_to_buffer(Y, U, V, "I420"), cv2.COLOR_YUV2BGR_I420))
    f = [rng.uniform(0.5, 2.0) for _ in range(B)]
    num = [(b * 3) % (rows + 1) for b in range(B)]
    num[33] = 0
    lines = rng.uniform(-1e3, 1e3, (B, rows, 9))
    for b, (h, w) in enumerate(sizes):
        lines[b, :num[b]] = random_lines(rng, num[b], h * f[b], w * f[b])
    desc = [d for fr in frames for d in yuv420_descriptor(fr)]
    buf, where, status = run_kernel("ctpn_line_crops_yuv420_u8", desc, sizes, f, lines, num, Hc)
    check_against_oracle(buf, where, status, bgr, lines, num, f, Hc)


# ---- the engine ---------------------------------------------------------------------------------------------------------

def check_source_crops(results, sources_bgr, Hc=32, plain=None):
    """Every result (lines, f, crops, widths[, resized]): crops equal cv2.warpAffine of the source with lines / f, zeros
    past the widths; lines and f equal those of the crop_height=None call `plain`.  Returns the number of lines."""
    total = 0
    for i, r in enumerate(results):
        lines, f, crops, widths = r[:4]
        if plain is not None:
            assert np.array_equal(plain[i][0], lines) and plain[i][1] == f
        m = len(lines)
        assert crops.is_cuda and crops.dtype == torch.uint8 and widths.dtype == np.int64
        assert np.array_equal(widths, crop.crop_widths(source_lines(lines, f), Hc))
        assert tuple(crops.shape) == (m, Hc, int(widths.max()) if m else 0, 3)
        c = crops.cpu().numpy()
        for j in range(m):
            assert np.array_equal(c[j, :, :widths[j]], cv2_source_crop(sources_bgr[i], lines[j], f, Hc)), (i, j)
            assert (c[j, :, widths[j]:] == 0).all()
        total += m
    return total


@pytest.mark.parametrize("mode", ["H", "O"])
def test_list_call_on_host_arrays(engine, images, mode):
    from ctpn_b200 import frontend_plan
    assert {p.dtype for p in frontend_plan(images)} == {"|u1", "<f4"}           # uint8 and float32-blob batches
    plain = engine.detect_lines_images(images, cfg=LOW, mode=mode)
    got = engine.detect_lines_images(images, cfg=LOW, mode=mode, crop_height=32, crop_from="source")
    assert check_source_crops(got, images, plain=plain) > 0
    rgb = [np.ascontiguousarray(im[:, :, ::-1]) for im in images[:6]]
    got = engine.detect_lines_images(rgb, cfg=LOW, mode=mode, crop_height=48, crop_from="source", channels="RGB", max_batch=4)
    assert check_source_crops(got, images[:6], Hc=48, plain=plain[:6]) > 0


@pytest.mark.parametrize("layouts", [BGR_LAYOUTS, RGB_LAYOUTS], ids=["bgr", "rgb"])
def test_list_call_on_tensors(engine, images, layouts):
    tensors, channels = device_list(images, layouts)
    plain = engine.detect_lines_images(images, cfg=LOW, mode="O")
    got = engine.detect_lines_images(tensors, cfg=LOW, mode="O", crop_height=32, crop_from="source", channels=channels,
                                     max_batch=7)
    assert check_source_crops(got, images, plain=plain) > 0


@pytest.mark.parametrize("layout", ["NV12", "I420"])
def test_list_call_on_frames(engine, layout):
    ph = video_photos(6)
    frames = [device_frame(*p, layout, seed=i) for i, (_, p) in enumerate(ph)]
    plain = engine.detect_lines_images([b for b, _ in ph], cfg=LOW)
    got = engine.detect_lines_images(frames, cfg=LOW, crop_height=32, crop_from="source")
    assert check_source_crops(got, [b for b, _ in ph], plain=plain) > 0


def test_at_f_1_source_crops_are_canvas_crops(engine, images):
    """resize=False, and 600 x 900 photos (already at the scale): f is 1, resize_im copies the image, and the crops agree
    bit for bit."""
    from oracle import synth
    ims = [im for im in images if min(im.shape[:2]) >= 200][:6]
    ims_600 = [synth.make_image(1700 + i, 600, 900) for i in range(3)]
    for batch, kw in ((ims, dict(resize=False)), (ims_600, {})):
        canvas = engine.detect_lines_images(batch, cfg=LOW, crop_height=32, **kw)
        source = engine.detect_lines_images(batch, cfg=LOW, crop_height=32, crop_from="source", **kw)
        assert sum(len(r[0]) for r in source) > 0
        for c, s in zip(canvas, source):
            assert c[1] == s[1] == 1.0 and np.array_equal(c[0], s[0]) and np.array_equal(c[3], s[3])
            assert torch.equal(c[2], s[2])


def test_the_calls_check_crop_from(engine, images):
    with pytest.raises(ValueError, match="crop_from must be"):
        engine.detect_lines_images(images[:1], crop_height=32, crop_from="canvas")
    with pytest.raises(ValueError, match="needs a crop_height"):
        engine.detect_lines_images(images[:1], crop_from="source")
    with pytest.raises(ValueError, match="needs a crop_height"):
        engine.stream_lines_images(iter(images[:1]), crop_from="source")


def same_crop_results(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert len(x) == len(y), i
        assert np.array_equal(x[0], y[0]) and x[1] == y[1] and np.array_equal(x[3], y[3]), i
        assert torch.equal(x[2], y[2]), i


def distinct_photos(n):
    """n photos of different content in several sizes, camera-size ones among them (compacted uploads without source
    crops)."""
    from oracle import synth
    sizes = [(480, 640), (1200, 1800), (300, 550), (2000, 1500), (600, 900), (3024, 4032)]
    return [synth.make_image(2000 + i, *sizes[i % len(sizes)]) for i in range(n)]


def test_stream_of_host_arrays_equals_the_list_call(engine):
    """max_batch 4 over 24 distinct photos: at least 6 batches, so each of the three source buffers is reused while the
    crop of the batch before is still to run."""
    ims = distinct_photos(24)
    want = engine.detect_lines_images(ims, cfg=LOW, mode="O", crop_height=32, crop_from="source", max_batch=4)
    assert check_source_crops(want, ims) > 0
    got = list(engine.stream_lines_images(iter(ims), cfg=LOW, mode="O", crop_height=32, crop_from="source", max_batch=4,
                                          window=8))
    same_crop_results(got, want)


def test_stream_of_tensors_and_frames_equals_the_list_call(engine):
    ims = distinct_photos(20)
    want = engine.detect_lines_images(ims, cfg=LOW, crop_height=32, crop_from="source", max_batch=4)

    def tensors():             # the stream holds the only references
        for i, im in enumerate(ims):
            t, ch = device_list([im], RGB_LAYOUTS[i % 3:] + RGB_LAYOUTS[:i % 3])
            yield t[0]
    got = list(engine.stream_lines_images(tensors(), cfg=LOW, crop_height=32, crop_from="source", max_batch=4, window=8,
                                          channels="RGB"))
    same_crop_results(got, want)
    ph = video_photos(20)
    want = engine.detect_lines_images([b for b, _ in ph], cfg=LOW, crop_height=32, crop_from="source", max_batch=4)
    assert check_source_crops(want, [b for b, _ in ph]) > 0
    frames = (device_frame(*p, ("NV12", "I420")[i % 2], seed=i) for i, (_, p) in enumerate(ph))
    got = list(engine.stream_lines_images(frames, cfg=LOW, crop_height=32, crop_from="source", max_batch=4, window=8))
    same_crop_results(got, want)


def test_crops_outlive_a_stream_closed_after_its_first_result(engine):
    ims = distinct_photos(12)
    want = engine.detect_lines_images(ims, cfg=LOW, crop_height=32, crop_from="source", max_batch=2)
    for kind in ("host", "tensor"):
        src = iter(ims) if kind == "host" else (torch.from_numpy(im).cuda() for im in ims)
        gen = engine.stream_lines_images(src, cfg=LOW, crop_height=32, crop_from="source", max_batch=2, window=4)
        kept = [next(gen)]
        gen.close()
        junk = [torch.full((1 << 24,), 0x3C, dtype=torch.uint8, device="cuda") for _ in range(8)]   # reuse freed blocks
        del junk
        same_crop_results(kept, want[:1])


def test_census():
    """The torch.profiler census of tests/source_crops_cases.py, in a process of its own (see test_line_crops_gpu.py)."""
    cmd = [sys.executable, "-m", "pytest", "-q", "-s", "-p", "no:cacheprovider", "-m", "gpu",
           os.path.join(HERE, "source_crops_cases.py") + "::test_census"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, cwd=os.path.dirname(HERE))
    assert p.returncode == 0 and " passed" in p.stdout and "failed" not in p.stdout, \
        "stdout:\n%s\nstderr:\n%s" % (p.stdout[-4000:], p.stderr[-2000:])
