"""Engine-level checks of photos already in device memory, run one test per process by tests/test_device_images_gpu.py
(this file is not collected by a plain pytest run: its name does not start with test_).  The raw-photo calls on CUDA
tensors return what they return on host copies, bit for bit; device-input streams equal the list calls, keep the tensors
a caller dropped and follow torch's stream rule; mixed inputs are refused as specified.  Each runs in a fresh process so
that the engines, streams and worker threads it creates leave nothing behind in the test session's process, where other
tests count kernels with torch.profiler.

    python -m pytest -q tests/device_images_cases.py::test_mixed_inputs_are_refused_and_the_engine_goes_on
"""
import numpy as np
import pytest
import torch

from device_image_checks import BGR_LAYOUTS, RGB_LAYOUTS, device_list, photos as make_photos
from oracle import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def weights():
    return synth.make_weights(0)


@pytest.fixture(scope="module")
def photos():
    return make_photos()


def same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert len(x) == len(y), i
        for u, v in zip(x, y):
            if isinstance(u, np.ndarray):
                assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v), i
            else:
                assert u == v, i


# ---- the list calls ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["f16f8", "bf16x2"])
def test_list_calls_on_device_tensors_equal_host_copies(weights, photos, mode):
    from ctpn_b200 import Engine, frontend_plan
    eng = Engine(weights, mode=mode)
    plan = frontend_plan(photos)
    assert {p.dtype for p in plan} == {"|u1", "<f4"}       # batches with uint8 and with float32 blobs
    for resize in (True, False):
        want = eng.rois_images(photos, resize=resize, return_resized=True)   # f16f8: the first batch calibrates the scales
        assert sum(r[0].shape[0] > 0 for r in want) >= len(photos) // 2
        for layouts in (BGR_LAYOUTS, RGB_LAYOUTS):
            tensors, channels = device_list(photos, layouts)
            for max_batch in (1, 7, 32, 64):
                same(eng.rois_images(tensors, resize=resize, max_batch=max_batch, return_resized=True, channels=channels), want)
            same(eng.detect_images(tensors, resize=resize, max_batch=7, channels=channels),
                 eng.detect_images(photos, resize=resize, max_batch=7))
    tensors, channels = device_list(photos, RGB_LAYOUTS)
    rgb_host = [np.ascontiguousarray(im[:, :, ::-1]) for im in photos]
    same(eng.rois_images(rgb_host, channels="RGB", return_resized=True), eng.rois_images(photos, return_resized=True))
    for line_mode in ("H", "O"):
        lines = eng.detect_lines_images(photos, mode=line_mode, return_resized=True)
        assert sum(r[0].shape[0] for r in lines) > 0
        same(eng.detect_lines_images(tensors, mode=line_mode, return_resized=True, channels=channels, max_batch=7), lines)


# ---- the streams ---------------------------------------------------------------------------------------------------------

def test_streams_of_device_tensors_equal_the_list_calls(weights, photos):
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="f16f8")
    want = eng.rois_images(photos, return_resized=True)
    det = eng.detect_images(photos)
    lines = eng.detect_lines_images(photos, mode="O")
    for layouts in (BGR_LAYOUTS, RGB_LAYOUTS):
        tensors, channels = device_list(photos, layouts)
        for window, max_batch in ((1, 1), (7, 5), (64, 32)):
            kw = dict(window=window, max_batch=max_batch, channels=channels)
            same(list(eng.stream_rois_images(iter(tensors), return_resized=True, **kw)), want)
            same(list(eng.stream_images(iter(tensors), **kw)), det)
            same(list(eng.stream_lines_images(iter(tensors), mode="O", **kw)), lines)
    rgb_host = [np.ascontiguousarray(im[:, :, ::-1]) for im in photos]       # host RGB through the row-compacting pack
    same(list(eng.stream_rois_images(iter(rgb_host), return_resized=True, window=7, max_batch=5, channels="RGB")), want)


def test_the_stream_keeps_tensors_the_caller_dropped(weights, photos):
    """Each tensor is created, yielded and dropped by the generator, and the caching allocator is handed new work that
    would reuse a freed block at once; the results do not change."""
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="bf16x2")
    want = eng.rois_images(photos)
    junk = []

    def fresh():
        for im in photos:
            yield torch.from_numpy(np.ascontiguousarray(im[:, :, ::-1])).cuda()
            junk.append(torch.full((im.size,), 0x3C, dtype=torch.uint8, device="cuda"))
            if len(junk) > 3:
                junk.pop(0)

    for window, max_batch in ((4, 4), (16, 32)):
        same(list(eng.stream_rois_images(fresh(), window=window, max_batch=max_batch, channels="RGB")), want)


def test_images_written_just_before_the_call_on_the_current_stream(weights, photos):
    """No synchronise between the kernel that writes the images and the call: the engine's work follows it on the
    current stream (and on a side stream made current for both)."""
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="bf16x2")
    want = eng.rois_images(photos)
    masked = [torch.from_numpy(im ^ 0x5A).cuda() for im in photos]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    for stream in (torch.cuda.current_stream(), side):
        with torch.cuda.stream(stream):
            torch.cuda._sleep(20_000_000)                                 # the writes below start late
            ready = [torch.bitwise_xor(m, 0x5A) for m in masked]
            got = eng.rois_images(ready, max_batch=7)
            torch.cuda._sleep(20_000_000)
            ready2 = [torch.bitwise_xor(m, 0x5A) for m in masked]
            gen = eng.stream_rois_images(iter(ready2), max_batch=5, window=7)
            got2 = list(gen)
        same(got, want)
        same(got2, want)
        del ready, ready2


def test_mixed_inputs_are_refused_and_the_engine_goes_on(weights, photos):
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="bf16x2")
    want = eng.detect_images(photos[:12])
    tensors = [torch.from_numpy(im).cuda() for im in photos[:12]]
    for bad in (photos[:5] + tensors[5:12], tensors[:3] + photos[3:12]):
        for call in (eng.rois_images, eng.detect_images, eng.detect_lines_images):
            with pytest.raises(ValueError, match="not both"):
                call(bad)
    with pytest.raises(ValueError, match="must be HxWx3 uint8"):
        eng.rois_images(tensors[:3] + [tensors[3].float()])
    with pytest.raises(ValueError, match="channels"):
        eng.detect_images(tensors, channels="rgb")
    with pytest.raises(ValueError, match="channels"):
        eng.stream_images(iter(tensors), channels="BGRA")
    same(eng.detect_images(tensors), want)
    for first, rest in ((tensors, photos), (photos, tensors)):
        got = []
        with pytest.raises(ValueError, match="image 9 is a .* but the stream's first image is .*not both"):
            for r in eng.stream_images(iter(first[:9] + rest[9:12]), max_batch=4, window=6):
                got.append(r)
        same(got, want[:9])
        same(list(eng.stream_images(iter(first[:12]), max_batch=4, window=6)), want)
    same(eng.detect_images(tensors), want)
