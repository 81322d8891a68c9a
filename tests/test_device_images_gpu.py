"""GPU: photos already in device memory.  ctpn_resize_linear_u8_strided writes what ctpn_resize_linear_u8_ragged writes on
dense BGR copies, and what the oracle computes, for every layout a caller will have.  The engine-level cases -- the six
raw-photo calls on CUDA tensors against host copies, stream lifetime and ordering, mixed inputs -- the profiler census of
a device-input stream and the nvJPEG checks each run in a process of their own (tests/device_images_cases.py,
tests/device_image_checks.py): the engines, streams, worker threads and profiler sessions they create must leave nothing
behind in the test session's process, where other tests count kernels with torch.profiler."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from device_image_checks import BGR_LAYOUTS, RGB_LAYOUTS, device_list, on_device
from oracle import resize as R, synth

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# (h, w, f): strong downscales of odd sizes, exact 1/2 with odd sides (INTER_AREA), f = 1, an upscale
KERNEL_CASES = [(3024 // 2 + 1, 403, 0.198), (1001, 333, 0.3), (301, 203, 0.5), (1200, 900, 0.5), (600, 450, 1.0),
                (97, 55, 1.25)]


def run_checks(*args, timeout=900):
    """tests/device_image_checks.py in a process of its own (see there why): its JSON result, which must say ok."""
    cmd = [sys.executable, os.path.join(HERE, "device_image_checks.py")] + [str(a) for a in args]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout)
    lines = [l for l in p.stdout.strip().splitlines() if l.startswith("{")]
    assert lines, "no result line.\nstdout:\n%s\nstderr:\n%s" % (p.stdout[-2000:], p.stderr[-3000:])
    res = json.loads(lines[-1])
    print(" ".join(str(a) for a in args), "->", json.dumps(res))
    assert res["ok"] and p.returncode == 0, "%s\nstderr:\n%s" % (json.dumps(res), p.stderr[-2000:])
    return res


# ---- the kernel ---------------------------------------------------------------------------------------------------------

def run_strided(tensors, channels, cases, sentinel=0xA5):
    from ctpn_b200 import _native as N
    from ctpn_b200.engine import resize_strided
    fxy = np.array([[c[2], c[2]] for c in cases], np.float64)
    dst_hw = np.array([R.out_size(c[0], c[1], c[2], c[2]) for c in cases], np.int32)
    B, H, W = len(cases), int(dst_hw[:, 0].max()) + 3, int(dst_hw[:, 1].max()) + 5
    canvas = torch.full((B, H, W, 3), sentinel, dtype=torch.uint8, device="cuda")
    resize_strided(tensors, channels, fxy, dst_hw, canvas, N.stream_ptr())
    return canvas.cpu().numpy(), dst_hw


def run_dense(images, cases, sentinel=0xA5):
    from ctpn_b200 import _native as N
    flat = np.concatenate([im.ravel() for im in images])
    offs = np.cumsum([0] + [im.size for im in images[:-1]]).astype(np.int64)
    hwp = np.array([(c[0], c[1], c[1]) for c in cases], np.int32)
    fxy = np.array([[c[2], c[2]] for c in cases], np.float64)
    dst_hw = np.array([R.out_size(c[0], c[1], c[2], c[2]) for c in cases], np.int32)
    B, H, W = len(cases), int(dst_hw[:, 0].max()) + 3, int(dst_hw[:, 1].max()) + 5
    src = torch.from_numpy(flat).cuda()
    canvas = torch.full((B, H, W, 3), sentinel, dtype=torch.uint8, device="cuda")
    N.check(N.lib.ctpn_resize_linear_u8_ragged(N.ptr(src), flat.size, N.ptr(offs), N.ptr(hwp), N.ptr(fxy), N.ptr(dst_hw), B, 3,
                                               N.ptr(canvas), H, W, N.stream_ptr()), "ctpn_resize_linear_u8_ragged")
    return canvas.cpu().numpy()


@pytest.mark.parametrize("layout", BGR_LAYOUTS + RGB_LAYOUTS)
def test_strided_kernel_equals_the_dense_kernel_and_the_oracle(layout):
    images = [synth.make_image(940 + i, h, w) for i, (h, w, _) in enumerate(KERNEL_CASES)]
    tensors, channels = device_list(images, (layout,))
    got, dst_hw = run_strided(tensors, channels, KERNEL_CASES)
    want = run_dense(images, KERNEL_CASES)
    assert np.array_equal(got, want)                       # the padding too: the sentinel survives in both
    for b, (h, w, f) in enumerate(KERNEL_CASES):
        dh, dw = dst_hw[b]
        assert np.array_equal(got[b, :dh, :dw], R.resize_linear_u8(images[b], f)), (layout, b)
        assert (got[b, dh:] == 0xA5).all() and (got[b, :, dw:] == 0xA5).all(), (layout, b)


def test_strided_kernel_mixed_layouts_and_broadcast_strides():
    images = [synth.make_image(960 + i, h, w) for i, (h, w, _) in enumerate(KERNEL_CASES)]
    tensors = [on_device(im, BGR_LAYOUTS[i % 3])[0] for i, im in enumerate(images)]
    px = torch.tensor([[[10, 200, 37]]], dtype=torch.uint8, device="cuda")
    row = torch.from_numpy(images[1][:1].copy()).cuda()
    tensors[2] = px.expand(KERNEL_CASES[2][0], KERNEL_CASES[2][1], 3)                 # zero strides everywhere
    images[2] = np.broadcast_to(px.cpu().numpy(), images[2].shape).copy()
    tensors[1] = row.expand(KERNEL_CASES[1][0], KERNEL_CASES[1][1], 3)                # one row, repeated
    images[1] = np.broadcast_to(images[1][:1], images[1].shape).copy()
    got, _ = run_strided(tensors, "BGR", KERNEL_CASES)
    assert np.array_equal(got, run_dense(images, KERNEL_CASES))


# ---- the raw-photo calls, one process per case (tests/device_images_cases.py) -------------------------------------------

ENGINE_CASES = ["test_list_calls_on_device_tensors_equal_host_copies", "test_streams_of_device_tensors_equal_the_list_calls",
                "test_the_stream_keeps_tensors_the_caller_dropped", "test_images_written_just_before_the_call_on_the_current_stream",
                "test_mixed_inputs_are_refused_and_the_engine_goes_on"]


@pytest.mark.parametrize("case", ENGINE_CASES)
def test_engine_case(case):
    """One engine-level case of tests/device_images_cases.py in a process of its own."""
    cmd = [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
           os.path.join(HERE, "device_images_cases.py") + "::" + case]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, cwd=os.path.dirname(HERE))
    assert p.returncode == 0 and " passed" in p.stdout and "failed" not in p.stdout, \
        "stdout:\n%s\nstderr:\n%s" % (p.stdout[-4000:], p.stderr[-2000:])


def test_a_device_stream_uploads_the_sizes_only_and_reads_in_place():
    """torch.profiler census of a warm device-input stream: per batch one H2D of at most the sizes / im_info tail, one
    strided resize kernel, no device-to-device copy or torch copy kernel, and no stream or device synchronise."""
    res = run_checks("census")
    assert res["batches"] >= 4 and len(res["uploads"]) == res["batches"] == res["strided"]


# ---- torchvision's nvJPEG in front ------------------------------------------------------------------------------------

def test_nvjpeg_decoded_photos_give_the_results_of_their_pixels():
    pytest.importorskip("torchvision")
    run_checks("nvjpeg")


def test_demo_gpu_decode_writes_the_files_of_the_decoded_pixels(tmp_path):
    """ctpn/demo.py --batch 4 --device-frontend --gpu-decode [--stream] on JPEGs and one PNG == --device-frontend on PNGs of
    the pixels nvJPEG decoded (and of the PNG)."""
    pytest.importorskip("torchvision")
    from ctpn import demo
    run_checks("demo", tmp_path)
    with pytest.raises(SystemExit):
        demo.main(["--batch", "4", "--gpu-decode"])
