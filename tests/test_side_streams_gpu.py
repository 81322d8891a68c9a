"""GPU: Engine(streams=k), which splits a batch into k sub-batches on side streams (detect_packed), against streams=1, bit
for bit: rois_batch at batch 32 x 600x900, 5 (an uneven split at k = 2 and 3) and 1 (the CUDA-graph path of streams=1),
detect_ragged, rois_images and stream_rois_images, in bf16x2, bf16x3p and f16f8.  F16F8 calibrates its activation scales on
the first forward; with streams > 1 that forward must still see the whole batch (tests/side_stream_checks.py, in its own
process on the test library)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import synth

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# photos for the front-end calls: upscale, exact 1/2, float rescale, portrait, f = 1
PHOTO_SIZES = [(240, 400), (1200, 1800), (300, 550), (450, 300), (600, 900), (1000, 3000), (700, 500)]
RAGGED_SIZES = [(600, 900), (480, 640), (900, 600), (333, 517), (600, 900), (64, 96), (250, 700)]


def same(a, b, what):
    assert len(a) == len(b), what
    for i, (x, y) in enumerate(zip(a, b)):
        x, y = (x, y) if isinstance(x, tuple) else ((x,), (y,))
        for u, v in zip(x, y):
            if isinstance(u, np.ndarray):
                assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v), (what, i)
            else:
                assert u == v, (what, i)


@pytest.mark.parametrize("mode", ["bf16x2", "bf16x3p", "f16f8"])
def test_side_streams_equal_one_stream(mode):
    from ctpn_b200 import Engine
    w = synth.make_weights(0)
    engines = {k: Engine(w, mode=mode, streams=k) for k in (1, 2, 3)}
    batch = np.stack([synth.make_image(200 + i, 600, 900) for i in range(32)])
    ragged = [synth.make_image(240 + i, h, w_) for i, (h, w_) in enumerate(RAGGED_SIZES)]
    photos = [synth.make_image(260 + i, h, w_) for i, (h, w_) in enumerate(PHOTO_SIZES * 2)]
    try:
        calls = [("rois_batch B=32", lambda e: e.rois_batch(batch)),          # f16f8: the first call calibrates
                 ("rois_batch B=5", lambda e: e.rois_batch(batch[3:8])),
                 ("detect_ragged", lambda e: e.detect_ragged(ragged, max_batch=5)),
                 ("rois_images", lambda e: e.rois_images(photos, max_batch=6)),
                 ("stream_rois_images", lambda e: list(e.stream_rois_images(iter(photos), max_batch=6, window=9)))]
        # B = 1: streams=1 runs the first two calls eagerly, then captures and replays a CUDA graph
        calls += [("rois_batch B=1 call %d" % n, lambda e: e.rois_batch(batch[7:8])) for n in range(4)]
        for what, call in calls:
            want = call(engines[1])
            assert sum(len(r[0] if isinstance(r, tuple) else r) for r in want) > 0, what
            for k in (2, 3):
                same(call(engines[k]), want, (mode, k, what))
        assert engines[1]._graphs and all("graph" in g for g in engines[1]._graphs.values())
    finally:
        del engines
        torch.cuda.empty_cache()


def run_checks(*args, timeout=600):
    cmd = [sys.executable, os.path.join(HERE, "side_stream_checks.py")] + [str(a) for a in args]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=dict(os.environ, CTPN_B200_LIB="dbg"))
    lines = [l for l in p.stdout.strip().splitlines() if l.startswith("{")]
    assert lines, "no result line.\nstdout:\n%s\nstderr:\n%s" % (p.stdout[-2000:], p.stderr[-3000:])
    res = json.loads(lines[-1])
    print(" ".join(str(a) for a in args), "->", json.dumps(res))
    assert res["ok"] and p.returncode == 0, "%s\nstderr:\n%s" % (json.dumps(res), p.stderr[-2000:])
    return res


def test_f16f8_side_streams_calibrate_on_the_whole_batch():
    res = run_checks("calibration")
    assert res["precondition"] and [s["step"] for s in res["steps"]] == ["first call", "second call", "recalibrate", "load_weights"]
