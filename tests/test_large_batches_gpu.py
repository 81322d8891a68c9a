"""GPU: the largest batches the engine runs.  conv1_1 and conv1_2 at batch 32 x 1200x1600 (bench.py --config 4), where plane
offsets pass 2^31 elements and 2^32 bytes (tests/large_checks.py, in its own process); the BiLSTM where its row groups need a
second wave of clusters; the engine at config 4's real batch against single images and the float32 oracle; and 64-image
ragged batches of photos (rois_images, detect_lines_images, stream_rois_images with max_batch=64) against single images.
Where the device has too little free memory a test skips and says how much it needs."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import net_cpu, postproc, synth

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def run_script(script, *args, timeout=1200):
    """As test_kernel_variants_gpu.run_script, and a result {"skip": reason} skips the test with that reason."""
    cmd = [sys.executable, os.path.join(HERE, script)] + [str(a) for a in args]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout)
    lines = [l for l in p.stdout.strip().splitlines() if l.startswith("{")]
    assert lines, "no result line.\nstdout:\n%s\nstderr:\n%s" % (p.stdout[-2000:], p.stderr[-3000:])
    res = json.loads(lines[-1])
    print(" ".join(str(a) for a in args), "->", json.dumps(res))
    if res.get("skip"):
        pytest.skip(res["skip"])
    assert res["ok"] and p.returncode == 0, "%s\nstderr:\n%s" % (json.dumps(res), p.stderr[-2000:])
    return res


def require_memory(need, what):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    free, total = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("%s needs %.1f GB of device memory; %.1f GB of %.1f GB are free" % (what, need / 1e9, free / 1e9, total / 1e9))


# ---- conv1_1 / conv1_2 past 2^31 elements and 2^32 bytes ---------------------------------------------------------------

@pytest.mark.parametrize("mode", ["bf16", "f16f8"])
def test_conv1_at_batch_32_1200x1600(mode):
    res = run_script("large_checks.py", "conv", "--mode", mode)
    assert res["conv1_1_bytes"] > 1 << 33 and len(res["boundary_pixels"]) >= 6, res
    assert {b for b, _, _ in res["boundary_pixels"]} == {2, 8, 17}, res["boundary_pixels"]


# ---- BiLSTM past one wave ----------------------------------------------------------------------------------------------

def per_wave():
    """2-CTA clusters of each direction in one wave (csrc/bilstm.cu, as test_kernel_variants_gpu.bilstm_rows derives it)."""
    return max(torch.cuda.get_device_properties(0).multi_processor_count // 4, 1)


# R: just past one wave at RG = 40, a max_batch=64 ragged batch of 600x900-class blobs (64 x 37 rows), config 4 at batch 32
# (32 x 75 rows)
BILSTM_ROWS = ["one_wave_plus_1", 2368, 2400]


@pytest.mark.parametrize("planes", [2, 3])
@pytest.mark.parametrize("W", [100, 56])
@pytest.mark.parametrize("rows", BILSTM_ROWS)
def test_bilstm_two_waves(rows, W, planes):
    pw = per_wave()
    R = 40 * pw + 1 if rows == "one_wave_plus_1" else rows
    assert math.ceil(R / 40) > pw, (R, pw)
    run_script("gpu_checks.py", "bilstm", "--R", R, "--W", W, "--planes", planes)


# ---- the engine at config 4's batch --------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def weights():
    return synth.make_weights(0)


@pytest.fixture(scope="module")
def config4_images():
    return np.stack([synth.make_image(900 + i, 1200, 1600) for i in range(32)])


@pytest.fixture(scope="module")
def config4_oracle_31(weights, config4_images):
    """The float32 CPU oracle's 1000 proposals of image 31."""
    im = config4_images[31]
    blob = (im.astype(np.float32) - net_cpu.PIXEL_MEANS.astype(np.float64)).astype(np.float32)[None]
    ref = net_cpu.forward(blob, weights)
    want, _ = postproc.proposal_layer(ref["rpn_cls_prob_reshape"], ref["rpn_bbox_pred"], np.array([[1200, 1600, 1.0]], np.float32))
    assert want.shape[0] == 1000
    return want


@pytest.mark.parametrize("mode", ["f16f8", "bf16x2"])
def test_config4_batch_32(weights, config4_images, config4_oracle_31, mode):
    from ctpn_b200 import Engine
    from ctpn_b200 import _native as N
    from test_net_gpu import rows_matched
    eng = Engine(weights, mode=mode)
    B, H, W = config4_images.shape[:3]
    need = N.lib.ctpn_net_workspace_bytes(eng._net, B, H, W) + N.lib.ctpn_proposals_workspace_bytes(B, H // 16, W // 16, 12000) \
        + config4_images.nbytes + (1 << 30)
    require_memory(need, "the engine at 32 x 1200x1600 (%s)" % mode)
    info = np.array([[H, W, 1.0]] * B, np.float32)
    batch = eng.rois_batch(config4_images, info)          # f16f8: the first call calibrates on this batch
    torch.cuda.synchronize()
    print("%s: peak device memory %.1f GB" % (mode, torch.cuda.max_memory_allocated() / 1e9))
    for i in (0, 15, 31):                                 # the third single-image call runs as a CUDA graph
        single = eng.rois_batch(config4_images[i:i + 1], info[:1])[0]
        assert single.shape == batch[i].shape and np.array_equal(single, batch[i]), i
    frac = rows_matched(batch[31], config4_oracle_31)
    print("%s: image 31 reproduces %.4f of the oracle's rows" % (mode, frac))
    assert batch[31].shape[0] == 1000 and frac >= 0.995
    del eng


# ---- 64-image ragged batches of photos -----------------------------------------------------------------------------------

# landscape photos whose blob is the uint8 resize_im output (im_scale 1), 600 x 750..850: 40 of them
LANDSCAPE = [(300, 400), (450, 600), (200, 250), (600, 850), (240, 320), (500, 700), (360, 480), (600, 640)]
# landscape exact 1/2 (INTER_AREA), blobs 600x850 and 600x900: they sort to the end of the landscape batch
HALVES = [(1200, 1700), (1200, 1800), (1200, 1800), (1200, 1700)]
PORTRAIT = [(400, 300), (900, 600), (1800, 1200), (800, 600), (1000, 700), (640, 480)] * 2
# float32 blobs (im_scale != 1): both orientations
FLOAT = [(200, 600), (1000, 3000), (300, 1000), (600, 200), (3000, 1000), (1000, 300), (250, 900), (900, 250)]


@pytest.fixture(scope="module")
def photos64():
    sizes = LANDSCAPE * 5 + HALVES + PORTRAIT + FLOAT
    assert len(sizes) == 64
    order = np.random.RandomState(0).permutation(64)       # input order unrelated to the batches' order
    return [synth.make_image(1000 + i, *sizes[i]) for i in order]


def same(a, b, what):
    assert len(a) == len(b), what
    for i, (x, y) in enumerate(zip(a, b)):
        assert len(x) == len(y), (what, i)
        for u, v in zip(x, y):
            if isinstance(u, np.ndarray):
                assert u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v), (what, i)
            else:
                assert u == v, (what, i)


def test_photo_plan_has_a_batch_past_32_with_an_exact_half_in_its_upper_half(photos64):
    from ctpn_b200 import frontend_plan, ragged_plan
    plan = frontend_plan(photos64)
    batches = ragged_plan([p.blob for p in plan], [p.dtype for p in plan], 64)
    big = max(batches, key=lambda b: len(b[0]))[0]
    assert len(big) > 32
    assert [k for k, i in enumerate(big) if plan[i].f == 0.5 and k >= 32], [plan[i].f for i in big]
    assert {p.dtype for p in plan} == {"|u1", "<f4"} and len(batches) >= 4


@pytest.mark.parametrize("mode", ["f16f8", "bf16x2"])
def test_64_image_batches_equal_single_images(weights, photos64, mode):
    from ctpn_b200 import Engine
    eng = Engine(weights, mode=mode)
    require_memory(24 << 30, "a 64-photo batch (%s)" % mode)
    eng.rois_images(photos64[:8], max_batch=8)            # f16f8: calibrate before the batch composition differs
    want = eng.rois_images(photos64, max_batch=1)
    assert sum(r[0].shape[0] for r in want) > 0
    same(eng.rois_images(photos64, max_batch=64), want, "rois_images")
    same(list(eng.stream_rois_images(iter(photos64), max_batch=64)), want, "stream_rois_images")
    for line_mode in ("H", "O"):
        lines = eng.detect_lines_images(photos64, mode=line_mode, max_batch=1)
        assert sum(r[0].shape[0] for r in lines) > 0
        same(eng.detect_lines_images(photos64, mode=line_mode, max_batch=64), lines, ("detect_lines_images", line_mode))
    torch.cuda.synchronize()
    print("%s: peak device memory %.1f GB" % (mode, torch.cuda.max_memory_allocated() / 1e9))
    del eng
