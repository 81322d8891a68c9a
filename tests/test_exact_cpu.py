"""CPU: the exact-arithmetic cases of tests/exact_cases.py -- their preconditions and coverage hold on the small cases of the
table, and the bit-for-bit comparison rejects a reference with a term the kernels' float64 bounds could not see: the
i + j = 2 plane pairs of bf16x3, or one K = 32 slice of an e4m3 cross product of F16F8."""
import pytest
import torch

import exact_cases as E
from variant_checks import CONV_TOL

SMALL = {k: c for k, c in E.VARIANT_CASES.items() if E.macs(c) <= 4e8}


def _operands(case):
    return (E.f16f8_operands if case["kind"] == "conv_f16f8" else E.bf16_operands)(case)


def test_the_table_has_small_cases_of_every_kind():
    kinds = {(c["kind"], c["taps"], c["planes"], bool(c["flags"] & E.F_PROMOTE)) for c in SMALL.values()}
    assert {("conv_f16f8", 9, 2, False), ("conv_f16f8", 1, 2, False), ("conv", 9, 3, True), ("conv", 1, 3, True)} <= kinds
    assert {p for kind, _, p, _ in kinds if kind == "conv"} == {1, 2, 3}


@pytest.mark.parametrize("key", list(SMALL), ids=str)
def test_preconditions_and_coverage(key):
    case = SMALL[key]
    ops = _operands(case)
    bounds, bad = E.check_preconditions(case, ops)
    assert not bad, (bounds, bad)
    assert bounds["acc_units"] <= E.ACC_BOUND and bounds.get("cross_units", 0) <= E.CROSS_BOUND
    if case["flags"] & E.F_RELU:
        assert 0 < bounds["relu_clipped"] < 1
    miss, ntiles = E.coverage(case, ops)
    assert ntiles > 0 and not any(miss.values()), miss
    y = E.reference(case, ops)
    assert torch.equal(y.float().double(), y)                      # one float32 value per output


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("blob", [False, True])
def test_conv1_1_preconditions_and_coverage(planes, blob):
    ops = E.conv1_operands(2, 37, 45, blob=blob)
    bounds, bad, miss, ntiles, y = E.conv1_check(ops, planes)
    assert not bad and not any(miss.values()), (bounds, bad, miss)
    if planes == 2:      # both cross pairs carry non-zero terms: the residual planes of the 9-10-bit values
        Ap, Wp = E.conv1_terms(ops, 2)
        assert Ap[1].abs().sum() > 0 and Wp[1].abs().sum() > 0


def test_every_output_plane_is_checked_in_every_tile():
    """The wide bias channels give outputs 19 significant bits, so the third bf16 plane is non-zero in every tile; with
    small biases alone (|y| < 2^12) it would be zero everywhere and the precondition refuses the case."""
    case = E.VARIANT_CASES[(9, 0, 3, 128, 0, 0)]
    ops = E.bf16_operands(case)
    bounds, bad = E.check_preconditions(case, ops)
    assert not bad and bounds["zero_plane_tiles"] == [0, 0, 0]
    assert (E.split_planes(E.reference(case, ops).float(), 3)[2] != 0).any()
    narrow = dict(ops, bias=E._bias(torch.Generator().manual_seed(1), case["cout"]))
    _, bad = E.check_preconditions(case, narrow)
    assert any("output plane 2 is zero" in b for b in bad), bad


@pytest.mark.parametrize("shape,fill", [((1, 9, 6), 0.88), ((1, 37, 56), 0.85)])
def test_near_bound_cross_cases_reach_the_bound(shape, fill):
    """The two F16F8 cases that measure the e4m3 accumulator near CROSS_BOUND stay within it and come within 5 % of it."""
    case = E.f16f8(*shape, 512, 512, 9, E.F_RELU, cross_fill=fill)
    bounds, bad = E.check_preconditions(case, E.f16f8_operands(case))
    assert not bad and 0.95 * E.CROSS_BOUND <= bounds["cross_units"] <= E.CROSS_BOUND, bounds


def test_simt_pairs_are_exact_too():
    """ctpn_conv3x3_simt multiplies the plane sums (all P^2 pairs): the same operands stay within the bound."""
    case = E.VARIANT_CASES[(9, 0, 3, 64, 0, 0)]
    ops = E.bf16_operands(case)
    bounds, bad = E.check_preconditions(case, ops, pairs="all")
    assert not bad, (bounds, bad)
    miss, _ = E.coverage(case, ops, pairs="all")
    assert not any(miss.values()), miss


def _report(name, y, y_bad, tol):
    rel = (y_bad - y).abs().max().item() / y.abs().max().item()
    print("%s: max |error| %.3g of max |y|; the float64 bound %.0e %s it" % (name, rel, tol, "rejects" if rel > tol else "accepts"))


def _gaussian(case):
    """Operands drawn as tests/gpu_checks.py draws them (activations, He-scaled weights, residual planes)."""
    g = torch.Generator().manual_seed(0)
    x = torch.relu(torch.randn(case["B"], case["H"], case["W"], case["cin"], generator=g))
    w = torch.randn(case["taps"], case["cin"], case["cout"], generator=g) * (2.0 / (case["taps"] * case["cin"])) ** 0.5
    return x, w, (torch.randn(case["cout"], generator=g) * 0.1).double()


def test_exact_comparison_rejects_bf16x3_without_the_i_plus_j_2_pairs():
    case = E.VARIANT_CASES[(9, 0, 3, 64, 0, 0)]
    ops = E.bf16_operands(case)
    y = E.reference(case, ops)
    x, w = ops["x"], ops["w"]
    two = [(x[0], w[2], 1.0), (x[1], w[1], 1.0), (x[2], w[0], 1.0)]
    y_bad = E.post(case, E.preact(case, ops) - E.partial(two, case["taps"]))
    want, got = E.split_planes(y.float(), 3), E.split_planes(y_bad.float(), 3)
    assert not torch.equal(want.view(torch.int16), got.view(torch.int16))
    assert not torch.equal(y.float(), y_bad.float())
    # every output tile sees the change
    assert E.tiles_changed(case, y, y_bad).all()
    _report("exact operands, bf16x3 without x0.w2 + x1.w1 + x2.w0", y, y_bad, CONV_TOL[3])
    # for the record: on the operands of the float64 checks the same bug stays below their bound
    xg, wg, bg = _gaussian(case)
    ops = dict(x=E.split_planes(xg, 3).double(), w=E.split_planes(wg, 3).double(), bias=bg)
    x, w = ops["x"], ops["w"]
    two = [(x[0], w[2], 1.0), (x[1], w[1], 1.0), (x[2], w[0], 1.0)]
    _report("gaussian operands, bf16x3 without the i + j = 2 pairs", E.reference(case, ops),
            E.post(case, E.preact(case, ops) - E.partial(two, case["taps"])), CONV_TOL[3])


def test_exact_comparison_rejects_f16f8_without_one_e4m3_slice():
    from oracle import quant
    case = E.VARIANT_CASES[(9, 1, 2, 128, 0, 0)]
    ops = E.f16f8_operands(case)
    y = E.reference(case, ops)
    # value x residual, tap 4, channel block 3, second K = 32 half
    va = torch.zeros_like(ops["v_a"])
    c0 = 3 * 64 + 32
    va[..., c0:c0 + 32] = ops["v_a"][..., c0:c0 + 32]
    rw = torch.zeros_like(ops["r_w"])
    rw[4] = ops["r_w"][4]
    y_bad = E.post(case, E.preact(case, ops) - E.partial([(va, rw, ops["inv_cross"])], case["taps"]))
    assert not torch.equal(y.float(), y_bad.float())
    assert E.tiles_changed(case, y, y_bad).all()
    out_t = quant.pow2_floor(448.0 / y.abs().max().item()) / 2.0
    h, cross, _ = quant.quantize(y.float(), 2.0, out_t)
    h2, cross2, _ = quant.quantize(y_bad.float(), 2.0, out_t)
    assert not (torch.equal(h.view(torch.int16), h2.view(torch.int16)) and torch.equal(cross, cross2))
    _report("exact operands, F16F8 without one value x residual K = 32 slice (float32 output)", y, y_bad, 2e-5)
    # for the record, on the operands of the float64 checks (dequantised: inv_main = inv_cross = 1)
    xg, wg, bg = _gaussian(case)
    _, _, (ha, va, ra) = quant.quantize(xg, 1.0, quant.pow2_floor(448.0 / float(xg.abs().max())) / 2.0)
    _, _, (hw, vw, rw) = quant.quantize(wg, quant.pow2_floor(16384.0 / float(wg.abs().max())), quant.pow2_floor(448.0 / float(wg.abs().max())))
    ops = dict(h_a=ha, v_a=va, r_a=ra, h_w=hw, v_w=vw, r_w=rw, bias=bg, inv_main=1.0, inv_cross=1.0)
    va = torch.zeros_like(ops["v_a"])
    va[..., c0:c0 + 32] = ops["v_a"][..., c0:c0 + 32]
    rw = torch.zeros_like(ops["r_w"])
    rw[4] = ops["r_w"][4]
    _report("gaussian operands, F16F8 without that slice", E.reference(case, ops),
            E.post(case, E.preact(case, ops) - E.partial([(va, rw, 1.0)], case["taps"])), 2e-5)
