"""Engine-level checks of YUV 4:2:0 frames in device memory, run one test per process by tests/test_yuv_frames_gpu.py (this
file is not collected by a plain pytest run: its name does not start with test_).  The six raw-photo calls on frames
return what they return on the BGR tensors cv2.cvtColor gives for those frames, bit for bit; streams equal the list calls,
keep the planes a caller dropped and follow torch's stream rule; bad frames are refused before any device work; and a
torch.profiler census shows that no image byte crosses the bus.

    python -m pytest -q tests/yuv_frames_cases.py::test_transfer_census
"""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from yuv_frames import LAYOUTS, device_frame, frames_of, video_photos

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.make_weights(0)


@pytest.fixture(scope="module")
def photos():
    return video_photos()


def same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert len(x) == len(y), i
        for u, v in zip(x, y):
            if isinstance(u, np.ndarray):
                assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v), i
            else:
                assert u == v, i


def bgr_tensors(photos):
    return [torch.from_numpy(b).cuda() for b, _ in photos]


# ---- the list calls ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["f16f8", "bf16x2"])
def test_list_calls_on_frames_equal_the_converted_tensors(weights, photos, mode):
    from ctpn_b200 import Engine, frontend_plan
    eng = Engine(weights, mode=mode)
    bgr = bgr_tensors(photos)
    assert {p.dtype for p in frontend_plan(bgr)} == {"|u1", "<f4"}          # batches with uint8 and with float32 blobs
    frames = frames_of(photos)
    for resize in (True, False):
        want = eng.rois_images(bgr, resize=resize, return_resized=True)      # f16f8: the first batch calibrates the scales
        assert sum(r[0].shape[0] > 0 for r in want) >= len(photos) // 2
        for max_batch in (1, 7, 32, 64):
            same(eng.rois_images(frames, resize=resize, max_batch=max_batch, return_resized=True), want)
        same(eng.detect_images(frames, resize=resize, max_batch=7, return_resized=True),
             eng.detect_images(bgr, resize=resize, max_batch=7, return_resized=True))
    for line_mode in ("H", "O"):
        lines = eng.detect_lines_images(bgr, mode=line_mode, return_resized=True)
        assert sum(r[0].shape[0] for r in lines) > 0
        same(eng.detect_lines_images(frames, mode=line_mode, return_resized=True, max_batch=7), lines)


# ---- the streams ---------------------------------------------------------------------------------------------------------

def test_streams_of_frames_equal_the_list_calls(weights, photos):
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="f16f8")
    bgr = bgr_tensors(photos)
    want = eng.rois_images(bgr, return_resized=True)
    det = eng.detect_images(bgr)
    lines = eng.detect_lines_images(bgr, mode="O")
    frames = frames_of(photos)
    for window, max_batch in ((1, 1), (7, 5), (16, 3), (64, 32)):
        kw = dict(window=window, max_batch=max_batch)
        same(list(eng.stream_rois_images(iter(frames), return_resized=True, **kw)), want)
        same(list(eng.stream_images(iter(frames), **kw)), det)
        same(list(eng.stream_lines_images(iter(frames), mode="O", **kw)), lines)


def test_the_stream_keeps_frames_the_caller_dropped(weights, photos):
    """Each frame is created, yielded and dropped by the generator, and the caching allocator is handed new work that
    would reuse a freed block at once; the results do not change."""
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="bf16x2")
    want = eng.rois_images(bgr_tensors(photos))
    junk = []

    def fresh():
        for i, (bgr, p) in enumerate(photos):
            yield device_frame(*p, LAYOUTS[i % len(LAYOUTS)], seed=i)
            junk.append(torch.full((bgr.size,), 0x3C, dtype=torch.uint8, device="cuda"))
            if len(junk) > 3:
                junk.pop(0)

    for window, max_batch in ((4, 4), (16, 32)):
        same(list(eng.stream_rois_images(fresh(), window=window, max_batch=max_batch)), want)


def test_frames_written_just_before_the_call(weights, photos):
    """No synchronise between the kernel that writes the planes and the call: the engine's work follows it on the current
    stream (and on a side stream made current for both)."""
    from ctpn_b200 import Engine, YUV420
    eng = Engine(weights, mode="bf16x2")
    want = eng.rois_images(bgr_tensors(photos))
    masked = [YUV420(*(p ^ 0x5A for p in f)) for f in frames_of(photos)]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    for stream in (torch.cuda.current_stream(), side):
        with torch.cuda.stream(stream):
            torch.cuda._sleep(20_000_000)                                 # the writes below start late
            ready = [YUV420(*(torch.bitwise_xor(p, 0x5A) for p in m)) for m in masked]
            got = eng.rois_images(ready, max_batch=7)
            torch.cuda._sleep(20_000_000)
            ready2 = [YUV420(*(torch.bitwise_xor(p, 0x5A) for p in m)) for m in masked]
            got2 = list(eng.stream_rois_images(iter(ready2), max_batch=5, window=7))
        same(got, want)
        same(got2, want)
        del ready, ready2


def test_bad_frames_are_refused_and_the_engine_goes_on(weights, photos):
    from ctpn_b200 import Engine, YUV420
    eng = Engine(weights, mode="bf16x2")
    bgr = bgr_tensors(photos[:12])
    want = eng.detect_images(bgr)
    frames = frames_of(photos[:12])
    host = [b for b, _ in photos[:12]]
    odd = YUV420(frames[1].y[:-1], frames[1].u, frames[1].v)
    cpu_plane = YUV420(frames[2].y, frames[2].u.cpu(), frames[2].v)
    for call in (eng.rois_images, eng.detect_images, eng.detect_lines_images):
        for bad, match in ((frames[:5] + host[5:], "is a host image but image 0 is a YUV420 frame"),
                           (bgr[:3] + frames[3:], "is a YUV420 frame but image 0 is a CUDA tensor"),
                           (frames[:1] + [odd] + frames[2:], "image 1 is a 1079x1920 YUV420 frame; 4:2:0 frames have even sides"),
                           (frames[:2] + [cpu_plane], "image 2: YUV420 plane u is not a CUDA tensor")):
            with pytest.raises(ValueError, match=match):
                call(bad)
        with pytest.raises(ValueError, match="converts to BGR"):
            call(frames, channels="RGB")
    same(eng.detect_images(frames), want)
    for first, rest, kind in ((frames, host, "a host image"), (frames, bgr, "a CUDA tensor"), (bgr, frames, "a YUV420 frame")):
        got = []
        with pytest.raises(ValueError, match="image 9 is %s but the stream's first image is .*not both" % kind):
            for r in eng.stream_images(iter(first[:9] + rest[9:12]), max_batch=4, window=6):
                got.append(r)
        same(got, want[:9])
    got = []
    with pytest.raises(ValueError, match="image 7 is a 1079x1920 YUV420 frame"):
        for r in eng.stream_images(iter(frames[:7] + [odd] + frames[8:]), max_batch=4, window=6):
            got.append(r)
    same(got, want[:7])
    with pytest.raises(ValueError, match="converts to BGR"):
        list(eng.stream_rois_images(iter(frames), channels="RGB"))
    same(list(eng.stream_images(iter(frames), max_batch=4, window=6)), want)


# ---- the transfer census -------------------------------------------------------------------------------------------------

def test_transfer_census(weights, photos):
    """torch.profiler census of warm calls on frames: per batch of a list call three small H2D copies -- im_info, the blob
    sizes and the feature sizes, 28 bytes an image -- and per stream batch one H2D of its 28-byte-per-image tail (sizes and
    im_info); no image byte.  One YUV resize launch
    per batch of at most 32 frames, no strided or dense resize kernel, no device-to-device copy or torch copy kernel."""
    from torch.profiler import ProfilerActivity, profile, record_function
    from ctpn_b200 import Engine, frontend_plan, ragged_plan
    eng = Engine(weights, mode="f16f8")
    frames = frames_of(photos)
    plan = frontend_plan(frames)
    list_batches = ragged_plan([p.blob for p in plan], [p.dtype for p in plan], 32)
    stream_batches = sum(len(ragged_plan([p.blob for p in plan[k:k + 8]], [p.dtype for p in plan[k:k + 8]], 4))
                         for k in range(0, len(plan), 8))

    def runs():
        return eng.rois_images(frames), list(eng.stream_rois_images(iter(frames), max_batch=4, window=8))

    want = runs()                          # warm: calibration, workspaces, slot buffers
    torch.cuda.synchronize()
    # a short run goes first inside the profile: the profiler can lose the first device records after it starts
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        eng.rois_images(frames[:4])
        torch.cuda.synchronize()
        with record_function("yuv_list_run"):
            got_list = eng.rois_images(frames)
            torch.cuda.synchronize()
        with record_function("yuv_stream_run"):
            got_stream = list(eng.stream_rois_images(iter(frames), max_batch=4, window=8))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    same(got_list, want[0])
    same(got_stream, want[1])
    res = {}
    for name, batches in (("yuv_list_run", list_batches), ("yuv_stream_run", stream_batches)):
        span = next(e for e in events if e.get("name") == name and e.get("cat") == "user_annotation")
        t0, t1 = span["ts"], span["ts"] + span["dur"]
        inside = [e for e in events if e.get("ph") == "X" and t0 <= e.get("ts", -1) <= t1]
        copies = [e for e in inside if e.get("cat") == "gpu_memcpy"]
        uploads = [int(e.get("args", {}).get("bytes", -1)) for e in copies if "HtoD" in e["name"]]
        kernels = [e["name"] for e in inside if e.get("cat") == "kernel"]
        n = batches if isinstance(batches, int) else len(batches)
        res[name] = dict(batches=n, uploads=uploads, dtod=sum("DtoD" in e["name"] for e in copies),
                         yuv=sum("resize_linear_u8_yuv420" in k for k in kernels),
                         unwanted=sorted({k for k in kernels if "resize_linear_u8_ragged" in k or "resize_linear_u8_strided" in k
                                          or "copy_kernel" in k.lower()}))
    print(json.dumps(res))
    lst, st = res["yuv_list_run"], res["yuv_stream_run"]
    assert sum(lst["uploads"]) == 28 * len(frames) and len(lst["uploads"]) == 3 * lst["batches"]
    assert lst["yuv"] == sum(-(-len(i) // 32) for i, _ in list_batches) and lst["dtod"] == 0 and not lst["unwanted"]
    assert len(st["uploads"]) == st["batches"] and all(0 < b <= 28 * 4 for b in st["uploads"])
    assert st["yuv"] == st["batches"] and st["dtod"] == 0 and not st["unwanted"]
