"""GPU: the F16F8 arithmetic at power-of-two scales other than 1, at kernel level against the exact quantiser and float64,
at net level under power-of-two rescaling of consecutive layers, and with scales calibrated on one image and used on another.

A value is carried as h = fp16(a s) plus e4m3(a t) and e4m3((a s - h) 2^11 t / s) with per-tensor powers of two s and t
(csrc/common.cuh, oracle/quant.py).  The calibration picks s = 1 unless a layer's maximum exceeds 2^14, and the synthetic
weights never get there, so the s != 1 paths (the fp16 pre-scale of the output quantiser, inv_main != 1 / s_w, the
calibration's s < 1 rule and its retry, the debug taps' decode) run here.  Kernel cases run in their own process
(tests/f16f8_scale_checks.py) with a timeout, as in test_kernel_variants_gpu.py."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from test_kernel_variants_gpu import RELU, POOL, VARIANTS, key_id
from variant_checks import F_STACK_OUT as STACK_OUT
from variant_checks import parse_label

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
F16F8_KEYS = [k for k in VARIANTS if k[1]]


def run_checks(*args, timeout=300, env=None):
    cmd = [sys.executable, os.path.join(HERE, "f16f8_scale_checks.py")] + [str(a) for a in args]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=dict(os.environ, **(env or {})))
    lines = [l for l in p.stdout.strip().splitlines() if l.startswith("{")]
    assert lines, "no result line.\nstdout:\n%s\nstderr:\n%s" % (p.stdout[-2000:], p.stderr[-3000:])
    res = json.loads(lines[-1])
    print(" ".join(str(a) for a in args), "->", json.dumps(res))
    assert res["ok"] and p.returncode == 0, "%s\nstderr:\n%s" % (json.dumps(res), p.stderr[-2000:])
    return res


def variant_args(cmd, key):
    """VARIANTS[key] (a gpu_checks conv_f16f8 command line) as the same layer for f16f8_scale_checks.py `cmd`."""
    args = list(VARIANTS[key])
    assert args[0] == "conv_f16f8"
    return [cmd] + args[1:]


# ---- 1. the output quantiser at out_s != 1, bit for bit -----------------------------------------------------------------

@pytest.mark.parametrize("key", F16F8_KEYS, ids=key_id)
def test_output_quantiser_equals_oracle_bit_for_bit(key):
    """Pooled (quarter-lane), staged long-K (Cin >= 256, no pool) and plain epilogues: F16F8 planes at out_s in
    {2^-6, 2^-1, 2^5} and three out_t equal oracle.quant.quantize of the same kernel's float32 output, with fp16 and
    e4m3 saturation and subnormals all reached."""
    res = run_checks(*variant_args("outq", key))
    assert {parse_label(l) for l in res["labels"]} == {key}, res["labels"]


@pytest.mark.parametrize("B,H,W,cin,cout,flags", [
    (1, 16, 24, 128, 128, RELU),                    # plain epilogue of a 3x3 layer (Cin < 256, no pool)
    (2, 50, 70, 64, 64, RELU | POOL | STACK_OUT),   # pooled epilogue into a row-stacked output
    (2, 9, 6, 512, 512, RELU | STACK_OUT),          # staged epilogue into a row-stacked output
])
def test_output_quantiser_plain_and_row_stacked(B, H, W, cin, cout, flags):
    res = run_checks("outq", "--B", B, "--H", H, "--W", W, "--cin", cin, "--cout", cout, "--taps", 9, "--flags", flags)
    assert {parse_label(l) for l in res["labels"]} <= set(VARIANTS), res["labels"]


def test_conv1_1_output_quantiser_scale_equivariance():
    """ctpn_conv1_1_tc_f16f8 has no float32 output: out_s -> 2^k out_s with t fixed moves the fp16 plane by exactly 2^k and
    leaves both e4m3 copies alone wherever the fp16 values stay normal and unsaturated."""
    res = run_checks("conv1_eqv", "--B", 2, "--H", 37, "--W", 45)
    assert res["labels"] == []


# ---- 2. input scale s_in != 1 -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("key", F16F8_KEYS, ids=key_id)
def test_input_scale_is_exact(key):
    """The same input at s_in = 2^k (k = -8, -2, 4) with inv_main = 1 / (s_in s_w): the main products scale by exactly 2^k and
    the e4m3 bytes do not change, so the float32 output is bit-identical to s_in = 1 (and within 2e-5 of float64)."""
    res = run_checks(*variant_args("sin", key))
    assert {parse_label(l) for l in res["labels"]} == {key}, res["labels"]


# ---- 3. inputs beyond the calibrated range ------------------------------------------------------------------------------

BEYOND = [(1, 16, 8, 64, 64, 9, RELU | POOL), (1, 9, 6, 512, 512, 9, RELU), (1, 1, 2072, 512, 64, 1, 0)]


@pytest.mark.parametrize("B,H,W,cin,cout,taps,flags", BEYOND)
def test_inputs_beyond_e4m3_range_keep_fp16_accuracy(B, H, W, cin, cout, taps, flags):
    """t_in calibrated on max|x| / 16: e4m3 copies saturate 2..6 binades up, fp16 does not.  Every output stays within
    BEYOND_GAIN * conv(|x|, |w|) (about 2^-10: fp16 accuracy) + 2e-5 max|y| of float64 on the true values."""
    run_checks("beyond", "--B", B, "--H", H, "--W", W, "--cin", cin, "--cout", cout, "--taps", taps, "--flags", flags)


@pytest.mark.parametrize("B,H,W,cin,cout,taps,flags", BEYOND[:2])
def test_inputs_saturating_fp16_stay_finite(B, H, W, cin, cout, taps, flags):
    """s_in with max|x| s_in >= 2^17: the fp16 plane saturates too; the output must be finite (the error is printed)."""
    run_checks("beyond", "--B", B, "--H", H, "--W", W, "--cin", cin, "--cout", cout, "--taps", taps, "--flags", flags,
               "--fp16sat", 1)


# ---- 4. net level: power-of-two rescaling of consecutive layers ---------------------------------------------------------

CONVS = ["conv1_1", "conv1_2", "conv2_1", "conv2_2", "conv3_1", "conv3_2", "conv3_3", "conv4_1", "conv4_2", "conv4_3",
         "conv5_1", "conv5_2", "conv5_3", "rpn_conv/3x3"]
LSTM_KERNELS = ["lstm_o/bidirectional_rnn/fw/lstm_cell/kernel", "lstm_o/bidirectional_rnn/bw/lstm_cell/kernel"]
SCALES = [2.0 ** -16, 2.0 ** -6, 2.0 ** 6, 2.0 ** 12]
# the layer each pair's second member reads, as a debug tap (F16F8 scales are per layer output)
NEXT_TAP = {l: (CONVS[l + 1] + "+pool" if CONVS[l + 1] in ("conv1_2", "conv2_2", "conv3_3", "conv4_3") else CONVS[l + 1])
            for l in range(13)}
NEXT_TAP[13] = "xproj"


def rescaled(weights, l, c):
    """Layer l's weights and bias times c, and what reads its output times 1 / c: conv l + 1, or for rpn_conv/3x3 the
    x-rows (the first 512) of both LSTM kernels.  The network's function is unchanged (ReLU and max-pool commute with c > 0)."""
    w = dict(weights)
    w[CONVS[l] + "/weights"] = weights[CONVS[l] + "/weights"] * np.float32(c)
    w[CONVS[l] + "/biases"] = weights[CONVS[l] + "/biases"] * np.float32(c)
    if l < 13:
        w[CONVS[l + 1] + "/weights"] = weights[CONVS[l + 1] + "/weights"] * np.float32(1.0 / c)
    else:
        for k in LSTM_KERNELS:
            k2 = weights[k].copy()
            k2[:512] *= np.float32(1.0 / c)
            w[k] = k2
    return w


@pytest.fixture(scope="module")
def weights():
    from oracle import synth
    return synth.make_weights(0)


@pytest.fixture(scope="module")
def small_case(weights):
    import torch
    from oracle import net_cpu, synth
    im = synth.make_image(7, 96, 160)
    blob = (im.astype(np.float32) - net_cpu.PIXEL_MEANS.astype(np.float64)).astype(np.float32)[None]
    ref = net_cpu.forward(blob, weights, dtype=torch.float64)
    return torch.from_numpy(im[None]).cuda(), ref


@pytest.mark.parametrize("mode", ["bf16", "bf16x2", "bf16x3", "bf16x3p"])
def test_bf16_modes_are_exactly_scale_equivariant(weights, small_case, mode):
    """bf16 planes of c a are c times the planes of a, the wgmma products and the truncating float32 accumulation scale
    exactly and ReLU and pooling commute with c: the head tensors of every rescaled net equal the unscaled net's bit for bit.
    A mismatch means an absolute constant somewhere in the arithmetic."""
    import torch
    from ctpn_b200 import Engine
    im, _ = small_case
    eng = Engine(weights, mode=mode)
    cls0, box0 = (t.clone() for t in eng.forward_heads(im))
    bad = []
    for l in range(14):
        for c in SCALES:
            eng.load_weights(rescaled(weights, l, c))
            cls, box = eng.forward_heads(im)
            if not (torch.equal(cls, cls0) and torch.equal(box, box0)):
                bad.append((CONVS[l], c, float((cls - cls0).abs().max()), float((box - box0).abs().max())))
    assert not bad, bad


def test_f16f8_rescaled_nets_against_float64(weights, small_case):
    """F16F8 is bit-identical under the rescaling up to elements that are fp16 subnormals at one of the two scales.  Every
    rescaled net keeps its head logits within the bounds of test_f16f8_mode_head_error_over_several_images of the float64
    oracle.  For c >= 2^6 (no new fp16 subnormals; s < 1 at 2^12) the layer reading the rescaled output stays within 1e-5 of
    the unscaled net (measured: 0 except where the unscaled layer had fp16 subnormals), which pins inv_main / inv_cross at
    input scales s < 1; for c < 1 new fp16 subnormals cost ~1e-5 there."""
    from ctpn_b200 import Engine
    im, ref = small_case
    eng = Engine(weights, mode="f16f8", keep_activations=True)
    cls0, box0 = (t.cpu().numpy() for t in eng.forward_heads(im))
    taps0 = {l: eng.tap(NEXT_TAP[l]).cpu().numpy() for l in range(14)}
    rows, bad = [], []
    for l in range(14):
        for c in SCALES:
            eng.load_weights(rescaled(weights, l, c))
            cls, box = (t.cpu().numpy() for t in eng.forward_heads(im))
            nxt = eng.tap(NEXT_TAP[l]).cpu().numpy()
            d_cls = float(np.abs(cls - ref["rpn_cls_score"]).max())
            d_box = float(np.abs(box - ref["rpn_bbox_pred"]).max())
            d_next = float(np.abs(nxt - taps0[l]).max() / np.abs(taps0[l]).max())
            d_c1 = float(max(np.abs(cls - cls0).max(), np.abs(box - box0).max()))
            rows.append((CONVS[l], c, d_cls, d_box, d_next, d_c1))
            if not (d_cls < 1e-3 and d_box < 2e-4 and (c < 1.0 or d_next <= 1e-5)):
                bad.append(rows[-1])
    for r in rows:
        print("%-13s c=2^%-3d head cls %.2e bbox %.2e | next layer vs c=1 %.2e | heads vs c=1 %.2e"
              % (r[0], int(np.log2(r[1])), r[2], r[3], r[4], r[5]))
    assert not bad, bad


def test_f16f8_calibrated_scales_follow_the_rule():
    """Test library: each layer's (s, t) is quant.activation_scales(amax), amax is within fp16 rounding of the float64
    oracle's layer maximum, every layer scaled by 2^12 calibrates to s < 1 and its debug tap decodes at that s.  At 2^13 and
    2^60 the layer's fp16 plane reaches 60000 at s = 1 and the calibration retries at 2^-8 steps; at 2^60 the maximum is at
    least 60000 * 2^40, so the plane still saturated at 2^-40 and the sixth retry (the last allowed) ran.  At 2^66 the maximum
    exceeds 65504 * 2^48 and the forward is refused with CtpnError."""
    from test_conv_gpu import DBG
    cases = ",".join("%d:12" % l for l in range(13)) + ",2:13,5:13,10:13,0:-16,4:-6,7:6,2:60,11:60,2:66,11:66"
    res = run_checks("net_scales", "--cases", cases, env=DBG, timeout=600)
    for c in res["cases"]:
        if c["layer"] is not None and 12 <= c["k"] <= 64:
            assert c["s"][c["layer"]] < 1.0, c
        if c["layer"] is not None and 13 <= c["k"] <= 64:
            assert c["amax"][c["layer"]] >= 60000.0, c                # reached only through the retry
        if c["layer"] is not None and c["k"] == 60:
            assert c["amax"][c["layer"]] * 2.0 ** -40 >= 60000.0, c    # saturated at s = 2^-40: six retries
    assert sum(c["k"] == 60 for c in res["cases"]) == 2 and sum(c["k"] > 64 for c in res["cases"]) == 2
    print("calibrated s per layer at c = 1:", res["cases"][0]["s"])


# ---- 5. calibrated on one image, run on another -------------------------------------------------------------------------

def conv_stack(im, weights, fp16_s=None):
    """conv1_1 .. rpn_conv/3x3 of oracle/net_cpu.py in float64 on the GPU for a uint8 image: each layer's output (after its
    pool), flattened NHWC.  fp16_s: plain fp16 arithmetic instead -- every layer after conv1_1 reads its input as
    fp16(x s) / s (saturating, s = fp16_s[l - 1]) and its weights as fp16(w s_w) / s_w, with products and sums exact.  That is
    what an F16F8 layer falls back to where its e4m3 copies saturate."""
    import torch
    import torch.nn.functional as F
    from oracle import net_cpu, quant
    blob = (im.astype(np.float32) - net_cpu.PIXEL_MEANS.astype(np.float64)).astype(np.float32)[None]
    x = torch.from_numpy(blob).cuda().double().permute(0, 3, 1, 2)
    outs = []
    for l, (name, _, _, pool) in enumerate(net_cpu.CONV_LAYERS):
        w = torch.from_numpy(weights[name + "/weights"]).cuda().double()
        if fp16_s is not None and l > 0:
            s = fp16_s[l - 1]
            x = (x * s).clamp(-65504.0, 65504.0).half().double() / s
            s_w = quant.weight_scales(float(w.abs().max()))[0]
            w = (w * s_w).half().double() / s_w
        b = torch.from_numpy(weights[name + "/biases"]).cuda().double()
        x = F.relu(F.conv2d(x, w.permute(3, 2, 0, 1), b, padding=1))
        if pool:
            x = F.max_pool2d(x, 2, 2)
        outs.append(x.permute(0, 2, 3, 1).reshape(-1))
    return outs


def low_contrast_image(seed, h, w):
    """Pixels within +-6 of the mean (ctpn/demo.py's grey warm-up, with a little noise)."""
    from oracle import net_cpu
    rs = np.random.RandomState(seed)
    mean = np.round(net_cpu.PIXEL_MEANS.reshape(3)).astype(np.int64)
    return np.clip(mean + rs.randint(-6, 7, size=(h, w, 3)), 0, 255).astype(np.uint8)


def stale_run(weights, im_cal, im):
    """An F16F8 engine calibrated on im_cal, then run on im: (rpn_conv/3x3 tap, heads, the engine), and the float64 conv stacks
    of both images."""
    import torch
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="f16f8", keep_activations=True)
    eng.forward_heads(torch.from_numpy(im_cal[None]).cuda())          # the first forward calibrates
    heads = [t.cpu().numpy() for t in eng.forward_heads(torch.from_numpy(im[None]).cuda())]
    return eng, eng.tap("rpn_conv/3x3").double(), heads, conv_stack(im_cal, weights), conv_stack(im, weights)


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


RESCALED_LAYER = 7          # conv4_1 x 2^12: s = 1/4 when calibrated on a photo


@pytest.mark.parametrize("which", ["synthetic", "s_below_1"])
def test_f16f8_other_photo_within_t_headroom(weights, which):
    """Calibrated on one photo, run on another of the same kind: every layer maximum stays within 4x (t's headroom), so
    nothing saturates and the run keeps the layer-wise bound of a net calibrated on the photo itself (5e-4 relative, as in
    test_net_gpu.py::test_layerwise_against_float64_oracle), also with a layer at s < 1."""
    from oracle import quant, synth
    w = weights if which == "synthetic" else rescaled(weights, RESCALED_LAYER, 2.0 ** 12)
    eng, got, _, cal, ref = stale_run(w, synth.make_image(8, 96, 160), synth.make_image(7, 96, 160))
    factors = [float(r.max() / c.max()) for r, c in zip(ref, cal)]
    s = [quant.activation_scales(float(c.max()))[0] for c in cal[:13]]
    print(which, "photo / calibration maxima:", ["%.2f" % f for f in factors], "s:", s)
    assert max(factors) <= 4.0
    assert (which == "synthetic") == all(v == 1.0 for v in s)
    err = rel(got, ref[13])
    print("rpn_conv/3x3 relative error %.2e" % err)
    assert err < 5e-4


@pytest.mark.parametrize("h,w", [(96, 160), (600, 900)])
def test_f16f8_low_contrast_calibration_falls_back_to_fp16(weights, h, w):
    """Calibrated on a low-contrast image, run on a photo: layer maxima 8x and more beyond the calibration, so the e4m3 copies
    of most elements saturate, while the fp16 plane (s = 1) does not.  The conv stack then keeps fp16 accuracy: its error is
    at most 1.5x that of plain fp16 arithmetic (conv_stack with fp16_s; the per-product bound of f16f8_scale_checks.py
    BEYOND_GAIN is 1.1x fp16's 2^-10)."""
    from oracle import quant, synth
    im = synth.make_image(7, h, w)
    eng, got, _, cal, ref = stale_run(weights, low_contrast_image(1, h, w), im)
    s = [quant.activation_scales(float(c.max()))[0] for c in cal[:13]]
    factors = [float(r.max() / c.max()) for r, c in zip(ref, cal)]
    print("photo / calibration maxima:", ["%.1f" % f for f in factors])
    assert s == [1.0] * 13 and max(float(r.max()) for r in ref[:13]) < 65504.0
    assert min(factors[:13]) > 8.0
    fp16_err = rel(conv_stack(im, weights, fp16_s=s)[13], ref[13])
    err = rel(got, ref[13])
    print("%dx%d rpn_conv/3x3 relative error: stale scales %.2e, plain fp16 %.2e" % (h, w, err, fp16_err))
    assert err <= 1.5 * fp16_err


def test_f16f8_fp16_saturation_past_65504_over_s(weights):
    """A layer calibrated to s < 1 on a low-contrast image, then run on a photo whose maximum there is more than 8x the
    calibration one: past 65504 / s the fp16 plane saturates together with the residual copy, so that layer's values are cut
    at 65504 / s + 448 / (2^11 t) and the error of those elements is their excess over the cut -- unbounded, as DESIGN.md
    section 5 states.  The heads stay finite."""
    import torch
    from oracle import net_cpu, quant, synth
    im, im_cal = synth.make_image(7, 96, 160), low_contrast_image(1, 96, 160)
    cal0, ref0 = conv_stack(im_cal, weights), conv_stack(im, weights)
    factors = [float(r.max() / c.max()) for r, c in zip(ref0[:13], cal0[:13])]
    L = int(np.argmax(factors[1:12])) + 1                                    # a conv layer followed by a conv layer
    c = 2.0 ** int(np.ceil(np.log2(32768.0 / float(cal0[L].max()))))        # calibration maximum in [2^15, 2^16)
    w = rescaled(weights, L, c)
    eng, got, heads, cal, ref = stale_run(w, im_cal, im)
    s, t = quant.activation_scales(float(cal[L].max()))
    cut = 65504.0 / s + 448.0 / (2048.0 * t)
    print("%s x 2^%d: calibration max %.4g (s = 2^%d), photo max %.4g (%.1fx), cut %.4g"
          % (net_cpu.CONV_LAYERS[L][0], int(np.log2(c)), float(cal[L].max()), int(np.log2(s)), float(ref[L].max()),
             factors[L], cut))
    assert s < 1.0 and factors[L] > 8.0 and float(ref[L].max()) > cut
    name = net_cpu.CONV_LAYERS[L][0] + ("+pool" if net_cpu.CONV_LAYERS[L][3] else "")
    tap = eng.tap(name).double()
    assert abs(float(tap.max()) - cut) <= 1e-6 * cut                        # cut exactly there
    over = ref[L] > 1.01 * cut                                               # (1 %: the stale layers' own error)
    assert bool(over.any())
    np.testing.assert_allclose(tap[over].cpu().numpy(), cut, rtol=1e-6)
    excess = float((ref[L] - cut).max())
    max_err = float((tap - ref[L]).abs().max())
    assert excess <= max_err * (1 + 1e-6) and max_err <= excess * (1 + 1e-3)   # the error is the excess over the cut
    assert all(np.isfinite(x).all() for x in heads)
    d = [float(np.abs(x - y).max()) for x, y in zip(heads, (lambda r: (r["rpn_cls_score"], r["rpn_bbox_pred"]))(
        net_cpu.forward((im.astype(np.float32) - net_cpu.PIXEL_MEANS.astype(np.float64)).astype(np.float32)[None], weights,
                        dtype=torch.float64)))]
    print("layer error %.3g (%.1f%% of its maximum); head max|diff| cls %.3g bbox %.3g" %
          (excess, 100.0 * excess / float(ref[L].max()), d[0], d[1]))
