"""GPU: every tensor-core convolution in exact integer arithmetic, bit for bit against float64 (tests/exact_cases.py).

The float64 checks of tests/test_kernel_variants_gpu.py and tests/test_conv_epilogue_gpu.py hold each kernel to a bound just
above its own rounding, so a term smaller than that (the i + j = 2 plane pairs of bf16x3, one e4m3 slice of F16F8, the third
output plane) is invisible to them.  Here the operands are integers whose sums every accumulator holds exactly, so each
output has one correct float32 value and any dropped, doubled or misplaced tap, channel slice, plane pair or cross MMA --
in any tile, since the coverage check proves every term reaches every output tile -- fails the case.

Cases: one per conv_tc instantiation (the keys and shapes of VARIANTS, with the label asserted), the handoff shapes of
tests/test_conv_epilogue_gpu.FLOAT64_CASES (many tiles per CTA, odd multicast pairs, BN 64 / 128 / 256, taps = 1 GEMMs),
promoted bf16x3p at many tiles, pooling at odd edges, row-stacked input and output, conv1_1 (planes 1 and 2, uint8 + LUT and
float blob, F16F8 output), the SIMT reference kernel of the test library and the bf16 weight packer, and two F16F8 cases
whose e4m3 cross sums come within a few percent of the 2^12 bound.  Cases run in their own processes (tests/exact_checks.py)
with a timeout, so a faulting kernel fails one test instead of the session.  On one H100
(700 W limit) the module takes about 7 minutes; small cases share a process, since most of their time is its start-up."""
import json
import os
import subprocess
import sys

import pytest

import exact_cases as E
from test_conv_epilogue_gpu import FLOAT64_CASES
from test_kernel_variants_gpu import STACK_SHAPES, VARIANTS, key_id
from variant_checks import parse_label

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
DBG = {"CTPN_B200_LIB": "dbg"}     # tests/_native/libctpn_b200_dbg.so: the SIMT reference kernels
RELU, POOL, PROMOTE, STACK_IN, STACK_OUT = E.F_RELU, E.F_POOL, E.F_PROMOTE, E.F_STACK_IN, E.F_STACK_OUT


def run_exact(*args, timeout=600, env=None):
    """One case, or several separated by "+" in one process (the result then holds each case's under "cases")."""
    cmd = [sys.executable, os.path.join(HERE, "exact_checks.py")] + [str(a) for a in args]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=dict(os.environ, **(env or {})))
    lines = [l for l in p.stdout.strip().splitlines() if l.startswith("{")]
    assert lines, "no result line.\nstdout:\n%s\nstderr:\n%s" % (p.stdout[-2000:], p.stderr[-3000:])
    res = json.loads(lines[-1])
    print(" ".join(str(a) for a in args), "->", json.dumps(res))
    assert res["ok"] and p.returncode == 0, "%s\nstderr:\n%s" % (json.dumps(res), p.stderr[-2000:])
    assert res["mismatches"] == 0 and res["uncovered"] == 0
    return res


def _without_xscale(args):
    args = list(args)
    if "--xscale" in args:
        i = args.index("--xscale")
        del args[i:i + 2]
    return args


# ---- one case per instantiation ------------------------------------------------------------------------------------------

def test_exact_cases_cover_exactly_the_variant_table():
    """A new conv_tc instantiation (a new VARIANTS row) fails here until it has an exact case at its shape."""
    assert set(E.VARIANT_CASES) == set(VARIANTS)
    for key, case in E.VARIANT_CASES.items():
        assert [str(a) for a in E.argv(case)] == [str(a) for a in _without_xscale(VARIANTS[key])], key


def _batch(cases):
    """Command line running the cases one after the other in one process."""
    args = []
    for c in cases:
        args += (["+"] if args else []) + list(c)
    return args


# Small cases share one process (most of a small case's time is the process start-up); the others run one per process.
SMALL_KEYS = [k for k, c in E.VARIANT_CASES.items() if E.macs(c) <= 4e8]
LARGE_KEYS = [k for k in E.VARIANT_CASES if k not in SMALL_KEYS]


@pytest.mark.parametrize("key", LARGE_KEYS, ids=key_id)
def test_variant_exact(key):
    res = run_exact(*E.argv(E.VARIANT_CASES[key]))
    assert {parse_label(l) for l in res["labels"]} == {key}, res["labels"]


def test_small_variants_exact():
    res = run_exact(*_batch(E.argv(E.VARIANT_CASES[k]) for k in SMALL_KEYS))
    assert len(res["cases"]) == len(SMALL_KEYS)
    for key, r in zip(SMALL_KEYS, res["cases"]):
        assert {parse_label(l) for l in r["labels"]} == {key}, (key, r["labels"])


# ---- tile ordering: many tiles per CTA, multicast pairs, epilogue handoff ------------------------------------------------

@pytest.mark.parametrize("case", list(FLOAT64_CASES))
def test_handoff_shapes_exact(case):
    res = run_exact(*_without_xscale(FLOAT64_CASES[case]))
    assert res["labels"] and {parse_label(l) for l in res["labels"]} <= set(VARIANTS), res["labels"]


EXTRA = {
    # bf16x3p at many tiles per cluster, and the promoted GEMM at 518 tiles
    "bf16x3p_mc_many_pool": E.conv(1, 150, 225, 64, 128, 9, 3, RELU | POOL | PROMOTE),
    "bf16x3p_t1_many": E.conv(1, 1, 66304, 64, 128, 1, 3, PROMOTE),
    # pooling at odd edges: odd H and W, ragged tiles on both axes, a map of one pooled pixel
    "pool_odd_p2_mc": E.conv(2, 19, 21, 64, 128, 9, 2, RELU | POOL),
    "pool_odd_p1": E.conv(1, 17, 9, 128, 64, 9, 1, RELU | POOL),
    "pool_3x3_p3_promote": E.conv(1, 3, 3, 64, 64, 9, 3, RELU | POOL | PROMOTE),
    "pool_odd_f16f8": E.f16f8(1, 33, 17, 64, 128, 9, RELU | POOL),
    "pool_odd_f16f8_mc": E.f16f8(3, 21, 13, 128, 64, 9, RELU | POOL),
    # the e4m3 cross accumulator near its precondition bound: per-output cross sums up to 0.98 x CROSS_BOUND
    "f16f8_cross_near_bound": E.f16f8(1, 9, 6, 512, 512, 9, RELU, cross_fill=0.88),
    "f16f8_cross_near_bound_mc": E.f16f8(1, 37, 56, 512, 512, 9, RELU, cross_fill=0.85),
}


@pytest.mark.parametrize("name", list(EXTRA))
def test_promoted_and_odd_pool_exact(name):
    res = run_exact(*E.argv(EXTRA[name]))
    assert res["labels"] and {parse_label(l) for l in res["labels"]} <= set(VARIANTS), res["labels"]


# ---- row-stacked input and output ----------------------------------------------------------------------------------------

STACK_PLANES = [(2, 0), (3, 0), (1, 0), (3, 1), (2, 0)]     # (planes, promote) per STACK_SHAPES row


@pytest.mark.parametrize("i", range(len(STACK_SHAPES)), ids=["B%d_%dx%d_c%d-%d" % s for s in STACK_SHAPES])
def test_row_stacked_exact(i):
    """Stacked input with stacked output (image rows exact, pad rows zero), compact planes and float32 output."""
    B, H, W, cin, cout = STACK_SHAPES[i]
    planes, promote = STACK_PLANES[i]
    res = run_exact(*E.argv(E.conv(B, H, W, cin, cout, 9, planes, RELU | STACK_IN | STACK_OUT | (PROMOTE if promote else 0))))
    assert res["stacked_in"] and res["runs"]["stacked_pad_rows"]["mismatches"] == 0
    assert {parse_label(l) for l in res["labels"]} <= set(VARIANTS), res["labels"]


# ---- conv1_1 -------------------------------------------------------------------------------------------------------------

CONV1_CASES = [("conv1", B, H, W, planes, blob) for B, H, W, planes, blob in
                [(2, 37, 45, 1, 0), (2, 37, 45, 2, 0), (1, 120, 200, 2, 0), (2, 37, 45, 1, 1), (2, 37, 45, 2, 1)]] + \
               [("conv1_q", 2, 37, 45, None, blob) for blob in (0, 1)]


def test_conv1_1_exact():
    """ctpn_conv1_1_tc at planes 1 and 2 from a LUT and a float blob, and ctpn_conv1_1_tc_f16f8."""
    cases = [[cmd, "--B", B, "--H", H, "--W", W, "--blob", blob] + ([] if planes is None else ["--planes", planes])
             for cmd, B, H, W, planes, blob in CONV1_CASES]
    res = run_exact(*_batch(cases))
    assert len(res["cases"]) == len(CONV1_CASES) and all(r["labels"] == [] for r in res["cases"])


# ---- the SIMT reference kernel and the weight packer ---------------------------------------------------------------------

SIMT_KEYS = [(9, 0, 1, 64, 0, 0), (9, 0, 1, 256, 0, 0), (9, 0, 2, 128, 0, 0), (9, 0, 3, 64, 0, 0), (9, 0, 3, 64, 0, 1),
             (1, 0, 2, 64, 0, 0), (1, 0, 3, 64, 0, 0)]


def test_simt_reference_exact():
    """ctpn_conv3x3_simt multiplies the plane sums (every pair) with float32 FMAs: exact on the same operands."""
    res = run_exact(*_batch(E.argv(E.VARIANT_CASES[k]) + ["--impl", "simt"] for k in SIMT_KEYS), env=DBG)
    assert len(res["cases"]) == len(SIMT_KEYS) and all(r["labels"] == [] for r in res["cases"])


def test_pack_weights_bit_exact():
    run_exact("pack")
