"""The torch.profiler census of text-line crops, run in a process of its own by tests/test_line_crops_gpu.py (this file is
not collected by a plain pytest run: its name does not start with test_).  With crop_height the line calls make the same
uploads, downloads and host synchronises as without it, and one crop kernel runs per batch that has lines.

    python -m pytest -q -m gpu tests/line_crops_cases.py::test_transfer_census
"""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from device_image_checks import photos

pytestmark = pytest.mark.gpu
# as in tests/test_line_crops_gpu.py: score thresholds low enough that the synthetic weights give the photos lines
LOW = (0.05, 0.2, 50, 0.5, 0.5, 0.0, 0.0, 16, 2)
RUNS = ("list", "list_crops", "stream", "stream_crops")


def test_transfer_census():
    from torch.profiler import ProfilerActivity, profile, record_function
    from ctpn_b200 import Engine, frontend_plan, ragged_plan
    from oracle import synth
    eng = Engine(synth.make_weights(0), mode="bf16x2")
    images = photos(16)
    plan = frontend_plan(images)
    batches = len(ragged_plan([p.blob for p in plan], [p.dtype for p in plan], 32))
    runs = {"list": lambda: eng.detect_lines_images(images, cfg=LOW),
            "list_crops": lambda: eng.detect_lines_images(images, cfg=LOW, crop_height=32),
            "stream": lambda: list(eng.stream_lines_images(iter(images), cfg=LOW, max_batch=4, window=8)),
            "stream_crops": lambda: list(eng.stream_lines_images(iter(images), cfg=LOW, max_batch=4, window=8, crop_height=32))}
    for fn in runs.values():               # warm: workspaces, slot buffers, pinned buffers
        fn()
    torch.cuda.synchronize()
    # one profiler session; a short run goes first inside it: the profiler can lose the first device records after it starts
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        eng.detect_lines_images(images[:1], cfg=LOW)
        torch.cuda.synchronize()
        for name in RUNS:
            with record_function(name):
                runs[name]()
                torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    res = {}
    for name in RUNS:
        span = next(e for e in events if e.get("name") == name and e.get("cat") == "user_annotation")
        t0, t1 = span["ts"], span["ts"] + span["dur"]
        inside = [e for e in events if e.get("ph") == "X" and t0 <= e.get("ts", -1) <= t1]
        copies = [e for e in inside if e.get("cat") == "gpu_memcpy"]
        res[name] = dict(h2d=sorted(int(e.get("args", {}).get("bytes", -1)) for e in copies if "HtoD" in e["name"]),
                         d2h=sorted(int(e.get("args", {}).get("bytes", -1)) for e in copies if "DtoH" in e["name"]),
                         syncs=sum("Synchronize" in e.get("name", "") for e in inside if e.get("cat") == "cuda_runtime"),
                         crops=sum("line_crops" in e["name"] for e in inside if e.get("cat") == "kernel"),
                         kernels=sum(e.get("cat") == "kernel" for e in inside))
    print(json.dumps(res))
    assert all(r["kernels"] > 0 for r in res.values()), res            # the session recorded device activity
    for a, b in (("list", "list_crops"), ("stream", "stream_crops")):
        assert res[a]["h2d"] == res[b]["h2d"] and res[a]["d2h"] == res[b]["d2h"] and res[a]["syncs"] == res[b]["syncs"], (a, res)
        assert res[a]["crops"] == 0 and 0 < res[b]["crops"]
    assert res["list_crops"]["crops"] <= batches
