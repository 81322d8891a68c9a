"""GPU: the wgmma implicit-GEMM convolution (ctpn_conv3x3) and the float32 SIMT reference
(ctpn_conv3x3_simt) against a float64 torch conv2d evaluated on exactly the operand values the
bf16 planes carry.  Each case runs in its own process (tests/gpu_checks.py) with a timeout so a
faulting kernel fails one test instead of the session."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
RELU, POOL, F32 = 1, 2, 4


DBG = {"CTPN_B200_LIB": "dbg"}     # tests/_native/libctpn_b200_dbg.so: SIMT references, tuning / ablation switches


def run_check(*args, timeout=300, env=None):
    cmd = [sys.executable, os.path.join(HERE, "gpu_checks.py")] + [str(a) for a in args]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=dict(os.environ, **(env or {})))
    lines = [l for l in p.stdout.strip().splitlines() if l.startswith("{")]
    assert lines, "no result line.\nstdout:\n%s\nstderr:\n%s" % (p.stdout[-2000:], p.stderr[-3000:])
    res = json.loads(lines[-1])
    print(" ".join(str(a) for a in args), "->", json.dumps(res))
    assert res["ok"] and p.returncode == 0, "%s\nstderr:\n%s" % (json.dumps(res), p.stderr[-2000:])
    return res


def conv_args(B, H, W, cin, cout, taps, planes, flags, impl="tc", seed=0):
    return ["conv", "--B", B, "--H", H, "--W", W, "--cin", cin, "--cout", cout, "--taps", taps, "--planes", planes,
            "--flags", flags, "--impl", impl, "--seed", seed]


# (B, H, W, cin, cout, taps, planes, flags)
TC_CASES = [
    (1, 1, 128, 64, 64, 1, 1, F32),            # one tile, one k-block: the minimal tensor-core round trip
    (1, 1, 128, 64, 64, 1, 1, 0),              # bf16 plane output
    (1, 1, 300, 256, 128, 1, 2, F32),          # 1x1 GEMM, ragged M, several k-blocks, 3 plane pairs
    (1, 8, 16, 64, 64, 9, 1, RELU | F32),      # one 8x16 patch, all 9 taps, zero halo on every side
    (2, 37, 56, 128, 128, 9, 2, RELU),         # conv5-sized ragged map, batch 2
    (1, 37, 56, 512, 512, 9, 1, RELU),         # K = 4608, BN = 256, two N tiles
    (1, 37, 56, 512, 512, 9, 3, RELU),         # six plane pairs (float32-equivalent)
    (3, 75, 112, 64, 64, 9, 2, RELU | POOL),   # fused 2x2 max-pool, odd height (75 -> 37), > 148 tiles
    (2, 30, 45, 128, 256, 9, 1, RELU | POOL),  # pool with odd width
    (1, 150, 225, 64, 128, 9, 2, RELU),        # many tiles per CTA: pipeline phase wrap-around
    (1, 1, 2072, 512, 1024, 1, 2, F32),        # the BiLSTM x-projection GEMM of one 600x900 image
    (1, 1, 2072, 512, 64, 1, 2, F32),          # the heads GEMM
]


@pytest.mark.parametrize("case", TC_CASES, ids=lambda c: "B%d_%dx%d_c%d-%d_t%d_p%d_f%d" % c)
def test_conv_tcgen05(case):
    run_check(*conv_args(*case))


@pytest.mark.parametrize("case", [TC_CASES[4], TC_CASES[5], TC_CASES[7]], ids=lambda c: "B%d_%dx%d_c%d-%d_t%d_p%d_f%d" % c)
def test_conv_tcgen05_single_cta_variant(case):
    """3x3 layers default to 2-CTA clusters with multicast weight tiles; CTPN_TC_MCAST=0 (test library) is the one-CTA-per-tile variant."""
    run_check(*conv_args(*case), env=dict(DBG, CTPN_TC_MCAST="0"))


# (B, H, W, cin, cout, taps, flags, xscale)
F16F8_CASES = [
    (1, 8, 16, 64, 64, 9, RELU, 1.0),             # one tile
    (2, 37, 56, 128, 128, 9, RELU, 1.0),          # ragged conv5-sized map, 2-CTA multicast path
    (1, 37, 56, 512, 512, 9, RELU, 4.0),          # K = 4608, four N tiles
    (3, 75, 112, 64, 64, 9, RELU | POOL, 30.0),   # fused pool, BN = 64, large activations
    (1, 150, 225, 64, 128, 9, RELU, 0.05),        # many tiles per CTA, small activations
    (1, 1, 2072, 512, 1024, 1, 0, 1.0),           # 1x1 GEMM (no ReLU: signed outputs)
]


@pytest.mark.parametrize("case", F16F8_CASES, ids=lambda c: "B%d_%dx%d_c%d-%d_t%d_f%d_x%g" % c)
def test_conv_f16f8(case):
    """The 2-unit arithmetic (fp16 main + e4m3 cross terms) against float64 on the carried operand values; float32, F16F8
    and bf16x2 outputs; device weight packer bit-exact against the same rules in torch."""
    B, H, W, cin, cout, taps, flags, xs = case
    run_check("conv_f16f8", "--B", B, "--H", H, "--W", W, "--cin", cin, "--cout", cout, "--taps", taps, "--flags", flags, "--xscale", xs)


@pytest.mark.parametrize("B,H,W,cin,cout", [(3, 37, 56, 128, 128), (5, 9, 20, 64, 64), (2, 75, 40, 256, 128)])
def test_conv_row_stacked_batches(B, H, W, cin, cout):
    """CTPN_F_STACK_IN / _OUT: one tall image with zero pad rows between the images == the per-image layout, bit for bit."""
    run_check("conv_stack", "--B", B, "--H", H, "--W", W, "--cin", cin, "--cout", cout)


SIMT_CASES = [
    (1, 13, 17, 64, 64, 9, 2, RELU),
    (2, 20, 30, 64, 128, 9, 3, RELU | POOL),
    (1, 1, 200, 128, 64, 1, 1, F32),
]


@pytest.mark.parametrize("case", SIMT_CASES, ids=lambda c: "B%d_%dx%d_c%d-%d_t%d_p%d_f%d" % c)
def test_conv_simt_reference(case):
    run_check(*conv_args(*case, impl="simt"), env=DBG)


@pytest.mark.parametrize("R,W,planes", [(37, 56, 2), (5, 7, 3), (1184, 56, 1), (600, 100, 2)])
def test_bilstm_recurrence(R, W, planes):
    run_check("bilstm", "--R", R, "--W", W, "--planes", planes)


@pytest.mark.parametrize("B,H,W,planes,impl", [(2, 37, 45, 2, "tc"), (1, 16, 8, 1, "tc"), (1, 50, 70, 3, "tc"), (1, 600, 900, 2, "tc"),
                                               (2, 37, 45, 2, "simt"), (1, 50, 70, 3, "simt")])
def test_conv1_1(B, H, W, planes, impl):
    run_check("conv1", "--B", B, "--H", H, "--W", W, "--planes", planes, "--impl", impl, env=DBG if impl == "simt" else None)
