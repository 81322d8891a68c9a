"""The torch.profiler census of line crops out of the source images, run in a process of its own by
tests/test_source_crops_gpu.py (this file is not collected by a plain pytest run: its name does not start with test_).

  * A list call with crop_from="source" makes the same uploads, downloads and host synchronises as without crops.
  * A stream of host photos with source crops uploads every photo whole: no row maps, h * w * 3 bytes per photo plus the
    28-byte sizes and im_info tail -- although the camera photos among them would be compacted without source crops.
  * Streams of tensors and of frames upload their 28-byte tails only.
  * One crop launch per batch with lines; two for a YUV batch of more than 32 frames with lines in both halves.

    python -m pytest -q -m gpu tests/source_crops_cases.py::test_census
"""
import json
import os
import tempfile

import cv2
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
LOW = (0.05, 0.2, 50, 0.5, 0.5, 0.0, 0.0, 16, 2)


def census(runs):
    """{name: {h2d, d2h (sorted byte counts), syncs, strided, yuv, canvas (crop launches), kernels}} of each run, in one
    profiler session."""
    from torch.profiler import ProfilerActivity, profile, record_function
    for fn in runs.values():               # warm: workspaces, slot buffers, pinned buffers
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        torch.zeros(1, device="cuda").add_(1)       # the profiler can lose the first device records after it starts
        torch.cuda.synchronize()
        for name, fn in runs.items():
            with record_function(name):
                fn()
                torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    res = {}
    for name in runs:
        span = next(e for e in events if e.get("name") == name and e.get("cat") == "user_annotation")
        t0, t1 = span["ts"], span["ts"] + span["dur"]
        inside = [e for e in events if e.get("ph") == "X" and t0 <= e.get("ts", -1) <= t1]
        copies = [e for e in inside if e.get("cat") == "gpu_memcpy"]
        kernels = [e["name"] for e in inside if e.get("cat") == "kernel"]
        res[name] = dict(h2d=sorted(int(e.get("args", {}).get("bytes", -1)) for e in copies if "HtoD" in e["name"]),
                         d2h=sorted(int(e.get("args", {}).get("bytes", -1)) for e in copies if "DtoH" in e["name"]),
                         syncs=sum("Synchronize" in e.get("name", "") for e in inside if e.get("cat") == "cuda_runtime"),
                         strided=sum("line_crops_strided" in k for k in kernels),
                         yuv=sum("line_crops_yuv420" in k for k in kernels),
                         canvas=sum("line_crops_kernel" in k for k in kernels), kernels=len(kernels))
    return res


def test_census():
    from ctpn_b200 import Engine, YUV420, frontend_plan
    from ctpn_b200.engine import stream_layout, stream_windows
    from oracle import synth
    from yuv_frames import device_frame, video_photos
    eng = Engine(synth.make_weights(0), mode="bf16x2")
    sizes = [(480, 640), (3024, 4032), (300, 550), (2000, 1500), (600, 900), (1200, 1800)]
    ims = [synth.make_image(2100 + i, *sizes[i % len(sizes)]) for i in range(12)]
    tensors = [torch.from_numpy(im).cuda() for im in ims]
    ph = video_photos(8)
    frames = [device_frame(*p, "NV12", seed=i) for i, (_, p) in enumerate(ph)]
    same = [synth.make_image(2200 + i, 480, 640) for i in range(40)]         # one batch of 40 frames: two YUV chunks
    big = [YUV420.from_buffer(torch.from_numpy(cv2.cvtColor(im, cv2.COLOR_BGR2YUV_I420)).cuda(), "I420") for im in same]
    src = dict(crop_height=32, crop_from="source", cfg=LOW)
    out = {}
    runs = {
        "list": lambda: eng.detect_lines_images(ims, cfg=LOW, max_batch=4),
        "list_source": lambda: out.__setitem__("list_source", eng.detect_lines_images(ims, max_batch=4, **src)),
        "stream_host": lambda: out.__setitem__("stream_host", list(eng.stream_lines_images(iter(ims), max_batch=4, window=8,
                                                                                          **src))),
        "stream_tensors": lambda: list(eng.stream_lines_images(iter(tensors), max_batch=4, window=8, **src)),
        "stream_frames": lambda: list(eng.stream_lines_images(iter(frames), max_batch=4, window=8, **src)),
        "list_yuv40": lambda: out.__setitem__("list_yuv40", eng.detect_lines_images(big, max_batch=40, **src)),
    }
    res = census(runs)
    print(json.dumps(res))
    assert all(r["kernels"] > 0 for r in res.values()), res
    a, b = res["list"], res["list_source"]
    assert a["h2d"] == b["h2d"] and a["d2h"] == b["d2h"] and a["syncs"] == b["syncs"], res
    assert a["strided"] == a["canvas"] == 0 and b["canvas"] == 0
    plan = frontend_plan(ims)
    from ctpn_b200 import ragged_plan
    batches = ragged_plan([p.blob for p in plan], [p.dtype for p in plan], 4)
    with_lines = sum(any(len(out["list_source"][i][0]) for i in idxs) for idxs, _ in batches)
    assert b["strided"] == with_lines > 0, (b, with_lines)
    # the stream of host photos: whole images, no row maps, exactly stream_layout(compact_rows=False) per batch
    stream_batches = list(stream_windows(iter(ims), 8, 4, lambda im, i: (im, frontend_plan([im], first=i)[0])))
    want = sorted(stream_layout(sb.items, [im.shape[:2] for im in sb.images], compact_rows=False).total
                  for sb in stream_batches)
    assert res["stream_host"]["h2d"] == want, (res["stream_host"]["h2d"], want)
    assert sum(want) >= sum(im.size for im in ims)
    assert any(p.rows is not None for p in plan)               # a compacted upload would have been smaller
    assert res["stream_host"]["strided"] == sum(any(len(out["stream_host"][i][0]) for i in sb.idxs) for sb in stream_batches)
    for name in ("stream_tensors", "stream_frames"):
        assert all(n <= 28 * 4 and n % 28 == 0 for n in res[name]["h2d"]), (name, res[name])
        assert res[name]["canvas"] == 0 and res[name]["strided" if name == "stream_tensors" else "yuv"] > 0
    halves = [any(len(r[0]) for r in out["list_yuv40"][:32]), any(len(r[0]) for r in out["list_yuv40"][32:])]
    assert res["list_yuv40"]["yuv"] == sum(halves) and sum(halves) > 0, (res["list_yuv40"], halves)
    assert np.sum([len(r[0]) for r in out["list_yuv40"]]) > 0
