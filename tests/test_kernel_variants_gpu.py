"""GPU: every kernel instantiation the product library can dispatch, against float64 at kernel level.

conv_tc_run (csrc/conv_tc.cu) picks one of 32 instantiations conv_tc_kernel<BN, P, TAPS, MC, F8, PR> from the layer's
shape, plane count and flags.  VARIANTS holds one case per launch_bn call site, keyed by
(taps, f16f8, planes, BN, mc, promote), and every case asserts both its float64 bound (that of gpu_checks.py for its
kernel class) and that the kernel the profiler saw run is exactly its key.  The launch census runs the engine in every
arithmetic mode and fails on any conv_tc instantiation that is not in VARIANTS, so a new dispatch path fails the suite
until it has a kernel test.  The BiLSTM is run at every row-group size it can pick, conv1_1 in its F16F8-output and
float-blob forms, row-stacked batches on bf16 planes, and a batch of 32 600x900 images against single-image runs.

Kernel cases run in their own process (tests/variant_checks.py, tests/gpu_checks.py) with a timeout, so a faulting
kernel fails one test instead of the session."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from variant_checks import parse_label

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
RELU, POOL, F32, PROMOTE = 1, 2, 4, 64


def run_script(script, *args, timeout=300):
    cmd = [sys.executable, os.path.join(HERE, script)] + [str(a) for a in args]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout)
    lines = [l for l in p.stdout.strip().splitlines() if l.startswith("{")]
    assert lines, "no result line.\nstdout:\n%s\nstderr:\n%s" % (p.stdout[-2000:], p.stderr[-3000:])
    res = json.loads(lines[-1])
    print(" ".join(str(a) for a in args), "->", json.dumps(res))
    assert res["ok"] and p.returncode == 0, "%s\nstderr:\n%s" % (json.dumps(res), p.stderr[-2000:])
    return res


def conv(B, H, W, cin, cout, taps, planes, flags):
    """gpu_checks.cmd_conv: ctpn_conv3x3 on bf16 planes (flags may include CTPN_F_PROMOTE with planes = 3)."""
    return ("conv", "--B", B, "--H", H, "--W", W, "--cin", cin, "--cout", cout, "--taps", taps, "--planes", planes, "--flags", flags)


def f16f8(B, H, W, cin, cout, taps, flags, xscale):
    """gpu_checks.cmd_conv_f16f8: ctpn_conv3x3_f16f8 with float32, F16F8 and bf16x2 outputs."""
    return ("conv_f16f8", "--B", B, "--H", H, "--W", W, "--cin", cin, "--cout", cout, "--taps", taps, "--flags", flags,
            "--xscale", xscale)


# (taps, f16f8, planes, BN, mc, promote) -> a case that reaches exactly that instantiation in the product library, in the
# order of the launch_bn calls in conv_tc_run.  Without tuning variables BN is 256 for one plane and 128 otherwise, halved
# until it divides Cout; a 3x3 layer runs on 2-CTA clusters (mc) when it has at least two 16x8 pixel tiles; a promoted
# single-CTA 3x3 layer runs at BN = 64.  Image sizes below are those of the whole network's input.
VARIANTS = {
    # ---- F16F8: fp16 main + e4m3 cross terms ----
    (9, 1, 2, 128, 1, 0): f16f8(1, 75, 112, 256, 512, 9, RELU, 1.0),            # conv4_1 of 600x900
    (9, 1, 2, 64, 1, 0): f16f8(2, 50, 70, 64, 64, 9, RELU | POOL, 8.0),         # conv1_2 of a 50x70 batch, odd pooled width
    (9, 1, 2, 128, 0, 0): f16f8(1, 9, 6, 512, 512, 9, RELU, 2.0),               # conv5 of 150x100: one ragged tile
    (9, 1, 2, 64, 0, 0): f16f8(1, 16, 8, 64, 64, 9, RELU | POOL, 1.0),          # exactly one full tile, pooled
    (1, 1, 2, 128, 0, 0): f16f8(1, 1, 300, 256, 128, 1, 0, 1.0),                # ragged 1x1 GEMM, Cout 128
    (1, 1, 2, 64, 0, 0): f16f8(1, 1, 2072, 512, 64, 1, 0, 1.0),                 # heads-shaped GEMM
    # ---- bf16x3 with the promoted main accumulator ----
    (9, 0, 3, 128, 1, 1): conv(1, 75, 112, 128, 256, 9, 3, RELU | PROMOTE),     # conv3_1 of 300x450
    (9, 0, 3, 64, 1, 1): conv(1, 300, 450, 64, 64, 9, 3, RELU | POOL | PROMOTE),   # conv1_2 of 300x450
    (9, 0, 3, 64, 0, 1): conv(1, 16, 8, 512, 512, 9, 3, RELU | PROMOTE),        # conv5 of 256x128: one tile, K = 4608
    (1, 0, 3, 128, 0, 1): conv(1, 1, 2072, 256, 512, 1, 3, PROMOTE),            # FC of 600x900 (plane output)
    (1, 0, 3, 64, 0, 1): conv(1, 1, 2072, 512, 64, 1, 3, F32 | PROMOTE),        # heads of 600x900
    # ---- bf16 planes, 2-CTA multicast 3x3 ----
    (9, 0, 1, 256, 1, 0): conv(2, 19, 21, 256, 512, 9, 1, RELU | POOL),         # ragged tiles, odd pool, batch 2
    (9, 0, 1, 128, 1, 0): conv(1, 150, 225, 128, 128, 9, 1, RELU | POOL),       # conv2_2 of 300x450, odd pooled width
    (9, 0, 1, 64, 1, 0): conv(1, 300, 450, 64, 64, 9, 1, RELU | POOL),          # conv1_2 of 300x450
    (9, 0, 2, 128, 1, 0): conv(1, 37, 56, 512, 512, 9, 2, RELU),                # conv5 of 600x900
    (9, 0, 2, 64, 1, 0): conv(2, 50, 70, 64, 64, 9, 2, RELU | POOL),            # conv1_2 of a 50x70 batch
    (9, 0, 3, 128, 1, 0): conv(1, 75, 112, 256, 512, 9, 3, RELU),               # conv4_1 of 600x900
    (9, 0, 3, 64, 1, 0): conv(3, 75, 112, 64, 64, 9, 3, RELU | POOL),           # odd height (75 -> 37), > 148 tiles
    # ---- bf16 planes, single-CTA 3x3 (one 16x8 tile) ----
    (9, 0, 1, 256, 0, 0): conv(1, 13, 7, 256, 256, 9, 1, RELU | POOL),         # ragged tile, odd pool on both axes
    (9, 0, 1, 128, 0, 0): conv(1, 8, 8, 128, 128, 9, 1, RELU | POOL),           # conv2_2 of 16x16
    (9, 0, 1, 64, 0, 0): conv(1, 11, 5, 64, 64, 9, 1, RELU | F32),              # ragged tile, float32 output
    (9, 0, 2, 128, 0, 0): conv(1, 9, 6, 512, 512, 9, 2, RELU | POOL),           # conv5 of 150x100
    (9, 0, 2, 64, 0, 0): conv(1, 16, 8, 64, 64, 9, 2, RELU),                    # exactly one full tile
    (9, 0, 3, 128, 0, 0): conv(1, 12, 8, 256, 256, 9, 3, RELU | POOL),          # conv4_x-sized channels, one tile
    (9, 0, 3, 64, 0, 0): conv(1, 16, 8, 64, 64, 9, 3, RELU | POOL),             # conv1_2 of a 16x8 map
    # ---- bf16 planes, taps = 1 (x-projection, FC and heads GEMMs) ----
    (1, 0, 1, 256, 0, 0): conv(1, 1, 2072, 512, 1024, 1, 1, F32),               # x-projection of 600x900
    (1, 0, 1, 128, 0, 0): conv(1, 1, 333, 256, 128, 1, 1, 0),                   # ragged M, plane output
    (1, 0, 1, 64, 0, 0): conv(1, 1, 2072, 512, 64, 1, 1, F32),                  # heads of 600x900
    (1, 0, 2, 128, 0, 0): conv(1, 1, 2072, 256, 512, 1, 2, 0),                  # FC of 600x900 (plane output)
    (1, 0, 2, 64, 0, 0): conv(1, 1, 777, 512, 64, 1, 2, F32),                   # ragged heads GEMM
    (1, 0, 3, 128, 0, 0): conv(1, 1, 2072, 512, 1024, 1, 3, F32),               # x-projection of 600x900
    (1, 0, 3, 64, 0, 0): conv(1, 1, 2072, 512, 64, 1, 3, F32),                  # heads of 600x900
}


def key_id(k):
    return "t%d_%sp%d_bn%d%s%s" % (k[0], "f16f8_" if k[1] else "", k[2], k[3], "_mc" if k[4] else "", "_promote" if k[5] else "")


def test_variant_table_has_one_row_per_launch_site():
    assert len(VARIANTS) == 32
    assert sum(k[1] for k in VARIANTS) == 6 and sum(k[5] for k in VARIANTS) == 5
    for taps, f8, planes, bn, mc, pr in VARIANTS:
        assert not (mc and taps == 1) and not (f8 and (pr or planes != 2)) and not (pr and planes != 3)


@pytest.mark.parametrize("key", list(VARIANTS), ids=key_id)
def test_conv_tc_variant_against_float64(key):
    res = run_script("variant_checks.py", *VARIANTS[key])
    assert {parse_label(l) for l in res["labels"]} == {key}, res["labels"]


# ---- launch census ----------------------------------------------------------------------------------------------------

CENSUS_SHAPES = [(1, 600, 900), (4, 300, 300), (1, 16, 16), (1, 50, 70)]


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.make_weights(0)


def test_launch_census_every_engine_variant_has_a_kernel_test(weights):
    """Every conv_tc instantiation the engine launches, in every mode, at a bench-like shape, a stacked batch and maps of a
    single tile, must have its row in VARIANTS."""
    import torch
    from ctpn_b200 import Engine
    from ctpn_b200 import _native as N
    from oracle import synth
    from variant_checks import conv_tc_labels
    seen = {}
    try:
        for mode in ("bf16", "bf16x2", "bf16x3", "f16f8", "bf16x3p"):
            eng = Engine(weights, mode=mode)
            N.check(N.lib.ctpn_prof_enable(1), "ctpn_prof_enable")
            for B, H, W in CENSUS_SHAPES:
                ims = np.stack([synth.make_image(60 + i, H, W) for i in range(B)])
                eng.forward_heads(torch.from_numpy(ims).cuda())
            seen[mode] = {parse_label(l) for l in conv_tc_labels()}
            N.check(N.lib.ctpn_prof_enable(0), "ctpn_prof_enable")
            del eng
    finally:
        N.lib.ctpn_prof_enable(0)
    for mode, keys in seen.items():
        print(mode, sorted(key_id(k) for k in keys))
    missing = {mode: sorted(key_id(k) for k in keys - set(VARIANTS)) for mode, keys in seen.items()}
    assert not any(missing.values()), "conv_tc instantiations launched without a kernel test: %s" % missing
    assert all(seen.values())


# ---- BiLSTM ------------------------------------------------------------------------------------------------------------

def bilstm_rows():
    """R values that make ctpn_bilstm_recurrent (csrc/bilstm.cu) pick each row group RG in {4, 8, 16, 32, 40} on this device,
    each leaving a ragged last group, as [(R, RG)].  The kernel takes the smallest RG whose ceil(R / RG) clusters fit in one
    wave of SMs / 4 clusters per direction.  On 132 SMs: R = 37, 133, 265, 529, 1057 and 1184 (batch 32 x 600x900)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per_wave = max(sms // 4, 1)

    def rg_of(R):
        return next((rg for rg in (4, 8, 16, 32) if (R + rg - 1) // rg <= per_wave), 40)
    rows = [37, per_wave * 4 + 1, per_wave * 8 + 1, per_wave * 16 + 1, per_wave * 32 + 1, 1184]
    return [(R, rg_of(R)) for R in rows]


BILSTM_IDS = ["rg4", "rg8", "rg16", "rg32", "rg40", "rg40_batch32"]
# (row, W, planes): planes 2 runs the fast cell math, 3 the accurate one
BILSTM_CASES = [(i, 56, p) for i in range(6) for p in (2, 3)] + [(2, 56, 1), (3, 1, 2)]


@pytest.mark.parametrize("row,W,planes", BILSTM_CASES, ids=["%s_w%d_p%d" % (BILSTM_IDS[c[0]], c[1], c[2]) for c in BILSTM_CASES])
def test_bilstm_every_row_group(row, W, planes):
    rows = bilstm_rows()
    assert [rg for _, rg in rows] == [4, 8, 16, 32, 40, 40], rows
    R, rg = rows[row]
    assert R % rg, (R, rg)                  # a ragged last group
    run_script("gpu_checks.py", "bilstm", "--R", R, "--W", W, "--planes", planes)


# ---- conv1_1 -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,H,W", [(2, 37, 45), (1, 600, 900)])
def test_conv1_1_f16f8_output(B, H, W):
    res = run_script("variant_checks.py", "conv1_q", "--B", B, "--H", H, "--W", W)
    assert res["labels"] == []


@pytest.mark.parametrize("planes", [1, 2, 3])
def test_conv1_1_float_blob_input(planes):
    run_script("variant_checks.py", "conv1_f32", "--B", 2, "--H", 37, "--W", 45, "--planes", planes)


# ---- row-stacked batches on bf16 planes --------------------------------------------------------------------------------

STACK_SHAPES = [(3, 37, 56, 128, 128), (5, 9, 20, 64, 64), (2, 75, 40, 256, 128),
                (3, 13, 8, 64, 64),          # three stacked tiles: the last multicast pair is one tile twice
                (32, 37, 56, 512, 512)]      # conv5 of the batch-32 600x900 bench


@pytest.mark.parametrize("planes,promote", [(1, 0), (2, 0), (3, 0), (3, 1)], ids=["p1", "p2", "p3", "p3_promote"])
@pytest.mark.parametrize("B,H,W,cin,cout", STACK_SHAPES)
def test_row_stacked_planes_equal_plain_layout(B, H, W, cin, cout, planes, promote):
    res = run_script("variant_checks.py", "stack_planes", "--B", B, "--H", H, "--W", W, "--cin", cin, "--cout", cout,
                     "--planes", planes, "--promote", promote)
    assert {parse_label(l) for l in res["labels"]} <= set(VARIANTS), res["labels"]


# ---- bench-shape batch -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["f16f8", "bf16x2"])
def test_batch_32_600x900_equals_single_images(weights, mode):
    """Batch 32 x 600x900 runs the 1/16-scale layers row-stacked; images 0, 15 and 31 (first, middle, last of the stack) must
    give the same head tensors and proposals as single-image runs through the same engine, bit for bit."""
    import torch
    from ctpn_b200 import Engine
    from oracle import synth
    eng = Engine(weights, mode=mode)
    ims = np.stack([synth.make_image(100 + i, 600, 900) for i in range(32)])
    batch = eng.detect_batch(ims)                 # f16f8: the first call calibrates the activation scales on this batch
    cls_b, box_b = eng.forward_heads(torch.from_numpy(ims).cuda())
    for i in (0, 15, 31):
        c1, b1 = eng.forward_heads(torch.from_numpy(ims[i:i + 1]).cuda())
        assert torch.equal(c1[0], cls_b[i]) and torch.equal(b1[0], box_b[i]), i
        s, b = eng.detect(ims[i])
        np.testing.assert_array_equal(s, batch[i][0])
        np.testing.assert_array_equal(b, batch[i][1])
