"""GPU: YUV 4:2:0 video frames in device memory.  ctpn_resize_linear_u8_yuv420 writes what ctpn_resize_linear_u8_strided
writes on the BGR image cv2.cvtColor gives for the frame, and what oracle/resize.py and cv2.resize compute on it, for
every layout (tests/yuv_frames.py), at f = 1, exact 1/2, strong downscales, upscales and portrait frames, in batches on
both sides of the 32-frame launch chunk.  The engine-level cases -- the six raw-photo calls on frames against the same
calls on the converted BGR tensors, streams, lifetime, ordering, rejections and the transfer census -- each run in a
process of their own (tests/yuv_frames_cases.py), as tests/test_device_images_gpu.py runs its cases."""
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

from oracle import resize as R, yuv
from yuv_frames import LAYOUTS, device_frame, planes_of, random_planes

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# (h, w, f): 1080p and 4K at resize_im's factor, f = 1, exact 1/2 (INTER_AREA), an upscale, portrait, a thin strip
KERNEL_CASES = [(1080, 1920, 600 / 1080), (2160, 3840, 600 / 2160), (600, 800, 1.0), (1200, 1600, 0.5), (240, 400, 2.5),
                (1920, 1080, 600 / 1080), (34, 1002, 0.6)]


def case_planes(i, h, w):
    """Even cases: a synthetic photo's planes; odd cases: random planes (every conversion branch, saturation included)."""
    if i % 2:
        return random_planes(700 + i, h, w)
    from oracle import synth
    return planes_of(synth.make_image(700 + i, h, w))


def canvas_for(cases, sentinel=0xA5):
    dst_hw = np.array([R.out_size(h, w, f, f) for h, w, f in cases], np.int32)
    B, H, W = len(cases), int(dst_hw[:, 0].max()) + 3, int(dst_hw[:, 1].max()) + 5
    return torch.full((B, H, W, 3), sentinel, dtype=torch.uint8, device="cuda"), dst_hw


def run_yuv(frames, cases):
    from ctpn_b200 import _native as N
    from ctpn_b200.engine import resize_yuv420
    canvas, dst_hw = canvas_for(cases)
    resize_yuv420(frames, np.array([[f, f] for _, _, f in cases], np.float64), dst_hw, canvas, N.stream_ptr())
    return canvas.cpu().numpy(), dst_hw


def run_strided(bgrs, cases):
    from ctpn_b200 import _native as N
    from ctpn_b200.engine import resize_strided
    canvas, dst_hw = canvas_for(cases)
    resize_strided([torch.from_numpy(b).cuda() for b in bgrs], "BGR", np.array([[f, f] for _, _, f in cases], np.float64),
                   dst_hw, canvas, N.stream_ptr())
    return canvas.cpu().numpy()


@pytest.fixture(scope="module")
def kernel_planes():
    out = []
    for i, (h, w, f) in enumerate(KERNEL_CASES):
        Y, U, V = case_planes(i, h, w)
        bgr = yuv.yuv_to_bgr(Y, U, V)
        want = R.resize_linear_u8(bgr, f)
        cv = cv2.resize(cv2.cvtColor(yuv.planes_to_buffer(Y, U, V, "NV12"), cv2.COLOR_YUV2BGR_NV12), None, None, fx=f, fy=f,
                        interpolation=cv2.INTER_LINEAR)
        assert np.array_equal(want, cv), i           # the oracle chain is cv2's chain on this frame
        out.append(((Y, U, V), bgr, want))
    return out


@pytest.mark.parametrize("layout", LAYOUTS)
def test_yuv_kernel_equals_the_strided_kernel_the_oracle_and_cv2(layout, kernel_planes):
    frames = [device_frame(*p, layout, seed=i) for i, (p, _, _) in enumerate(kernel_planes)]
    got, dst_hw = run_yuv(frames, KERNEL_CASES)
    assert np.array_equal(got, run_strided([b for _, b, _ in kernel_planes], KERNEL_CASES))   # sentinel padding too
    for b, (_, _, want) in enumerate(kernel_planes):
        dh, dw = dst_hw[b]
        assert np.array_equal(got[b, :dh, :dw], want), (layout, b)
        assert (got[b, dh:] == 0xA5).all() and (got[b, :, dw:] == 0xA5).all(), (layout, b)


@pytest.mark.parametrize("B", [1, 7, 33, 64])
def test_batches_across_the_launch_chunk(B, kernel_planes):
    """B frames of every case and layout in turn: the 32-frame chunks write their own canvas slices."""
    small = [(h // 4 * 2, w // 4 * 2, f) for h, w, f in KERNEL_CASES]             # halved sides keep 64 frames quick
    cases = [small[i % len(small)] for i in range(B)]
    planes = [random_planes(900 + i, h, w) for i, (h, w, _) in enumerate(cases)]
    frames = [device_frame(*p, LAYOUTS[i % len(LAYOUTS)], seed=i) for i, p in enumerate(planes)]
    got, _ = run_yuv(frames, cases)
    assert np.array_equal(got, run_strided([yuv.yuv_to_bgr(*p) for p in planes], cases))


def test_a_plane_smaller_than_its_box_is_refused():
    """The C entry point checks each plane's box against its allocation: a V plane of 15 rows where the frame needs 16."""
    from ctpn_b200 import CtpnError, YUV420
    from ctpn_b200 import _native as N
    from ctpn_b200.engine import resize_yuv420
    f = YUV420.from_buffer(torch.full((48, 40), 16, dtype=torch.uint8, device="cuda"), "NV12")
    canvas = torch.full((1, 32, 40, 3), 7, dtype=torch.uint8, device="cuda")
    args = (np.array([[1.0, 1.0]]), np.array([[32, 40]], np.int32), canvas, N.stream_ptr())
    with pytest.raises(CtpnError, match="image 0: the V plane"):
        resize_yuv420([YUV420(f.y, f.u, torch.zeros(15, 20, dtype=torch.uint8, device="cuda"))], *args)
    assert int(canvas.ne(7).sum()) == 0
    resize_yuv420([f], *args)
    assert torch.equal(canvas[0].cpu(), torch.from_numpy(yuv.yuv_to_bgr(*[p.cpu().numpy() for p in f])))


# ---- the raw-photo calls, one process per case (tests/yuv_frames_cases.py) ------------------------------------------------

ENGINE_CASES = ["test_list_calls_on_frames_equal_the_converted_tensors", "test_streams_of_frames_equal_the_list_calls",
                "test_the_stream_keeps_frames_the_caller_dropped", "test_frames_written_just_before_the_call",
                "test_bad_frames_are_refused_and_the_engine_goes_on", "test_transfer_census"]


@pytest.mark.parametrize("case", ENGINE_CASES)
def test_engine_case(case):
    """One engine-level case of tests/yuv_frames_cases.py in a process of its own."""
    cmd = [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
           os.path.join(HERE, "yuv_frames_cases.py") + "::" + case]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, cwd=os.path.dirname(HERE))
    assert p.returncode == 0 and " passed" in p.stdout and "failed" not in p.stdout, \
        "stdout:\n%s\nstderr:\n%s" % (p.stdout[-4000:], p.stderr[-2000:])
