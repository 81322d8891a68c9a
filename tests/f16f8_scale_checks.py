#!/usr/bin/env python
"""Stand-alone GPU checks of the F16F8 arithmetic at power-of-two scales other than 1, run as subprocesses by
tests/test_f16f8_scales_gpu.py so that a faulting kernel fails one test instead of the session.  Each sub-command prints one
JSON line {"ok": bool, "labels": [...], ...} as its last line of stdout (labels: the conv_tc instantiations that ran, as in
tests/variant_checks.py).

    outq       ctpn_conv3x3_f16f8 with F16F8 output at out_s in {2^-6, 2^-1, 2^5} and three out_t: the planes must equal
               oracle.quant.quantize of the kernel's own float32 output (CTPN_F_OUT_F32) bit for bit
    conv1_eqv  ctpn_conv1_1_tc_f16f8 at out_s = 2^k: e4m3 value bytes identical, fp16 plane exactly 2^k x and residual bytes
               identical wherever both fp16 values are normal and unsaturated
    sin        the same layer input quantised at s_in = 2^k, k in {-8, -2, 4}, with inv_main = 1 / (s_in s_w): float32 output
               bit-identical to s_in = 1, and within 2e-5 * max|y| of float64
    beyond     inputs quantised with t_in calibrated on max|x| / 16 (e4m3 copies saturate, fp16 does not): per-element error
               within BEYOND_GAIN * conv(|x|, |w|) + 2e-5 * max|y| of float64 on the true values, and within 2e-5 * max|y|
               of float64 on the carried values (saturated copies included); with --fp16sat the fp16 plane saturates too and
               only finiteness is asserted
    net_scales a calibrated F16F8 net (test library: ctpn_net_f16f8_scales): scales equal quant.activation_scales(amax), amax
               within fp16 rounding of the float64 oracle's layer maximum, with layers rescaled by 2^k; a layer maximum
               beyond 65504 * 2^48 (k > 64 here) is refused

    python tests/f16f8_scale_checks.py outq --B 1 --H 16 --W 8 --cin 64 --cout 64 --taps 9 --flags 3
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT, os.path.join(ROOT, "text-detection-ctpn_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import variant_checks  # noqa: E402
from gpu_checks import F_F32, F_POOL, F_RELU  # noqa: E402
from variant_checks import F_STACK_OUT  # noqa: E402

OUT_S = (2.0 ** -6, 2.0 ** -1, 2.0 ** 5)
OUT_T = (2.0 ** -12, 2.0 ** -4, 2.0 ** 2)
S_IN_EXP = (-8, -2, 4)
# Per product a * w the kernel drops r_a * r_w and replaces r_a h_w + h_a r_w by e4m3 cross terms.  With |r| <= 2^-11 |x| (fp16
# rounding) and e4m3 rounding 2^-4, a saturated e4m3 copy of a (error <= |a|) and of r_a (error <= |r_a|) leave
#   |a - V_a| |r_w| + |V_a| |r_w - R_w| + |r_a| |h_w - V_w| + |r_a - R_a| |V_w|
#     <= 2^-11 |a||w| (1 + 2^-4 (1 + 2^-4) + (2^-4 + 2^-11) + (1 + 2^-4)) < 2^-11 * 2.19 |a||w|,
# i.e. fp16 accuracy (h_a h_w alone is within 2^-10 |a||w|).  Rounded up:
BEYOND_GAIN = 1.1 * 2.0 ** -10


def _layer(a, dev, wide_bias=False):
    """Input x (post-ReLU, zero or >= xscale 2^-5 so that x * 2^-8 stays normal fp16), weights, bias and the packed F16F8
    weights of a layer drawn as gpu_checks.cmd_conv_f16f8 draws them.  wide_bias: every fourth channel gets a bias of
    2^(-4..13) (fp16 and e4m3 saturation at the larger scales), every fourth a small negative one (values near 0)."""
    import torch
    from ctpn_b200 import _native as N
    from oracle import quant
    g = torch.Generator(device="cpu").manual_seed(a.seed)
    x = torch.relu(torch.randn(a.B, a.H, a.W, a.cin, generator=g)) * a.xscale
    x[x < a.xscale * 2.0 ** -5] = 0.0
    w = torch.randn(a.taps, a.cin, a.cout, generator=g) * (2.0 / (a.taps * a.cin)) ** 0.5
    b = torch.randn(a.cout, generator=g) * 0.1
    if wide_bias:
        b[1::4] = 2.0 ** torch.linspace(-4.0, 13.0, a.cout // 4)
        b[2::4] = -torch.rand(a.cout // 4, generator=g) * a.xscale
    s_w, t_w = quant.weight_scales(float(w.abs().max()))
    wp = torch.zeros(2 * a.cout * a.taps * a.cin * 2, dtype=torch.uint8, device=dev)
    N.check(N.lib.ctpn_pack_weights_f16f8(N.ptr(w.to(dev).contiguous()), a.taps, a.cin, a.cout, a.cout, s_w, t_w, N.ptr(wp),
                                          N.stream_ptr()), "pack")
    return x, w, b.to(dev), wp, s_w, t_w


def _packed_input(x, s, t, dev):
    """x quantised at (s, t) as the kernels' input planes on dev, and its dequantised (h, v8, r8) in float64"""
    import torch
    from oracle import quant
    h, cross, deq = quant.quantize(x, s, t)
    return torch.cat([h.view(torch.uint8).reshape(-1), cross.reshape(-1)]).to(dev), deq


def _run(a, inp, wp, bd, flags, inv_main, inv_cross, out_s, out_t, out):
    import torch
    from ctpn_b200 import _native as N
    N.check(N.lib.ctpn_conv3x3_f16f8(N.ptr(inp), N.ptr(wp), N.ptr(bd), N.ptr(out), a.B, a.H, a.W, a.cin, a.cout, a.taps, flags,
                                     inv_main, inv_cross, out_s, out_t, N.stream_ptr()), "conv_f16f8")
    torch.cuda.synchronize()
    return out


def _out_hw(a):
    return (a.H // 2, a.W // 2) if a.flags & F_POOL else (a.H, a.W)


def _ref64(a, xd, wd, bd, dev):
    """float64 conv (+bias, ReLU, pool) of NHWC x with [taps][Cin][Cout] w, as NHWC."""
    import torch
    k = 3 if a.taps == 9 else 1
    wr = wd.to(dev).double().permute(2, 0, 1).reshape(a.cout, k, k, a.cin).permute(0, 3, 1, 2)
    y = torch.nn.functional.conv2d(xd.to(dev).double().permute(0, 3, 1, 2), wr, None, padding=k // 2)
    if bd is not None:
        y = y + bd.double().view(1, -1, 1, 1)
    if a.flags & F_RELU:
        y = torch.relu(y)
    if a.flags & F_POOL:
        y = torch.nn.functional.max_pool2d(y, 2, 2)
    return y.permute(0, 2, 3, 1).contiguous()


def _quant_classes(v, s, t):
    """Counts of the format's edge cases among float32 values v quantised at (s, t): fp16 plane saturated / subnormal,
    e4m3 value copy saturated / subnormal, e4m3 residual copy saturated / subnormal."""
    import torch
    vs = (v.double() * s).abs()
    h = (v * s).clamp(-65504.0, 65504.0).to(torch.float16).float()
    r = ((v * s - h) * (2048.0 * t / s)).double().abs()
    vt = (v.double() * t).abs()
    return dict(h_sat=int((vs > 65504.0).sum()), h_sub=int(((vs > 0) & (vs < 2.0 ** -14)).sum()),
                v8_sat=int((vt > 448.0).sum()), v8_sub=int(((vt > 0) & (vt < 2.0 ** -6)).sum()),
                r8_sat=int((r > 448.0).sum()), r8_sub=int(((r > 0) & (r < 2.0 ** -6)).sum()))


def cmd_outq(a):
    import torch
    from oracle import quant
    dev = torch.device("cuda", 0)
    x, w, bd, wp, s_w, t_w = _layer(a, dev, wide_bias=True)
    s_in, t_in = quant.activation_scales(float(x.abs().max()))
    inp, _ = _packed_input(x, s_in, t_in, dev)
    inv_main, inv_cross = 1.0 / (s_in * s_w), 1.0 / (2048.0 * t_in * t_w)
    Ho, Wo = _out_hw(a)
    C = a.cout
    so = bool(a.flags & F_STACK_OUT)
    rows = Ho + 1 if so else Ho
    o32 = torch.full((a.B, Ho, Wo, C), float("nan"), dtype=torch.float32, device=dev)
    _run(a, inp, wp, bd, (a.flags & ~F_STACK_OUT) | F_F32, inv_main, inv_cross, 1.0, 1.0, o32)
    v = o32.cpu()
    res = dict(nan=int(torch.isnan(v).sum()), cases=[])
    classes = {}
    ok = res["nan"] == 0
    nel = a.B * rows * Wo * C
    for out_s in OUT_S:
        for out_t in OUT_T:
            oq = torch.full((nel * 4,), 0xAB, dtype=torch.uint8, device=dev)
            _run(a, inp, wp, bd, a.flags, inv_main, inv_cross, out_s, out_t, oq)
            oq = oq.cpu()
            h = oq[:nel * 2].view(torch.int16).view(a.B, rows, Wo, C)[:, :Ho]
            cr = oq[nel * 2:].view(a.B, rows, Wo, C // 64, 128)[:, :Ho]
            wh, wc, _ = quant.quantize(v, out_s, out_t)
            bad_h = int((h != wh.view(torch.int16)).sum())
            bad_v8 = int((cr[..., :64] != wc[..., :64]).sum())
            bad_r8 = int((cr[..., 64:] != wc[..., 64:]).sum())
            cls = _quant_classes(v, out_s, out_t)
            for k_, n_ in cls.items():
                classes[k_] = classes.get(k_, 0) + n_
            res["cases"].append(dict(out_s=out_s, out_t=out_t, bad_h=bad_h, bad_v8=bad_v8, bad_r8=bad_r8))
            ok = ok and bad_h == bad_v8 == bad_r8 == 0
    res["classes"] = classes
    covered = all(n > 0 for n in classes.values())
    res.update(ok=bool(ok and covered), covered=covered)
    print(json.dumps(res))
    return 0 if res["ok"] else 1


def cmd_conv1_eqv(a):
    """conv1_1 has no float32 output: with t fixed and out_s -> out_s * 2^k the e4m3 value bytes must not change; fp16 plane
    and residual bytes follow 2^k exactly on the elements whose fp16 values are normal and unsaturated at both scales."""
    import torch
    from ctpn_b200 import _native as N
    dev = torch.device("cuda", 0)
    rs = np.random.RandomState(a.seed)
    im = rs.randint(0, 256, size=(a.B, a.H, a.W, 3)).astype(np.uint8)
    w, b, lut = variant_checks._conv1_weights(rs)
    imd, wd, bd, lutd = (torch.from_numpy(z).to(dev) for z in (im, w, b, lut))
    nel = a.B * a.H * a.W * 64
    out_t = 2.0 ** -2

    def run(out_s):
        oq = torch.zeros(nel * 4, dtype=torch.uint8, device=dev)
        N.check(N.lib.ctpn_conv1_1_tc_f16f8(N.ptr(imd), 0, N.ptr(lutd), N.ptr(wd), N.ptr(bd), N.ptr(oq), a.B, a.H, a.W, out_s, out_t,
                                            N.stream_ptr()), "conv1_1_tc_f16f8")
        torch.cuda.synchronize()
        oq = oq.cpu()
        return oq[:nel * 2].view(torch.float16).view(-1, 64), oq[nel * 2:].view(-1, 128)
    h0, c0 = run(1.0)
    res = dict(cases=[])
    ok = bool(torch.isfinite(h0.float()).all())
    for k in (-16, -6, 3, 14):
        h1, c1 = run(2.0 ** k)
        a0, a1 = h0.float().abs(), h1.float().abs()
        # strictly above 2^-14: a subnormal y 2^k can round up to exactly 2^-14 on the subnormal grid
        both = (a0 > 2.0 ** -14) & (a0 < 65504.0) & (a1 > 2.0 ** -14) & (a1 < 65504.0)
        bad_v8 = int((c0[:, :64] != c1[:, :64]).sum())
        bad_h = int(((h1.double() != h0.double() * 2.0 ** k) & both).sum())
        bad_r8 = int(((c0[:, 64:] != c1[:, 64:]) & both.view(-1, 64)).sum())
        changed = int((~both & (h0 != 0)).sum())
        res["cases"].append(dict(k=k, compared=int(both.sum()), edge=changed, bad_h=bad_h, bad_v8=bad_v8, bad_r8=bad_r8))
        ok = ok and bad_h == bad_v8 == bad_r8 == 0 and int(both.sum()) > 0
    # the run at 2^14 must actually reach fp16 saturation (|y| > 4), the one at 2^-16 fp16 subnormals (|y| < 4)
    edges = {c["k"]: c["edge"] for c in res["cases"]}
    res["ok"] = bool(ok and edges[14] > 0 and edges[-16] > 0)
    print(json.dumps(res))
    return 0 if res["ok"] else 1


def cmd_sin(a):
    import torch
    from oracle import quant
    dev = torch.device("cuda", 0)
    x, w, bd, wp, s_w, t_w = _layer(a, dev)
    t_in = quant.activation_scales(float(x.abs().max()))[1]
    inv_cross = 1.0 / (2048.0 * t_in * t_w)
    Ho, Wo = _out_hw(a)
    outs, res, ok = {}, dict(cases=[]), True
    for k in (0,) + S_IN_EXP:
        s_in = 2.0 ** k
        inp, (xh, xv, xr) = _packed_input(x, s_in, t_in, dev)
        o32 = torch.full((a.B, Ho, Wo, a.cout), float("nan"), dtype=torch.float32, device=dev)
        _run(a, inp, wp, bd, a.flags | F_F32, 1.0 / (s_in * s_w), inv_cross, 1.0, 1.0, o32)
        outs[k] = o32
        # float64 on the carried values (gpu_checks.cmd_conv_f16f8)
        wt = w.permute(2, 0, 1).contiguous()
        _, _, (wh, wv, wr) = quant.quantize(wt, s_w, t_w)
        wh, wv, wr = (z.permute(1, 2, 0).contiguous() for z in (wh, wv, wr))
        a_ = argparse.Namespace(**{**vars(a), "flags": 0})
        y = _ref64(a_, xh, wh, None, dev) + _ref64(a_, xv, wr, None, dev) + _ref64(a_, xr, wv, None, dev)
        y = _finish(a, y, bd)
        scale = y.abs().max().item()
        err = (o32.double() - y).abs().max().item()
        same = bool(torch.equal(o32, outs[0]))
        res["cases"].append(dict(k=k, err=err, scale=scale, identical=same))
        ok = ok and err <= 2e-5 * scale and same and not bool(torch.isnan(o32).any())
    res["ok"] = bool(ok)
    print(json.dumps(res))
    return 0 if ok else 1


def _finish(a, y, bd):
    """bias, ReLU and pool on an NHWC float64 pre-activation"""
    import torch
    y = (y + bd.double()).permute(0, 3, 1, 2)
    if a.flags & F_RELU:
        y = torch.relu(y)
    if a.flags & F_POOL:
        y = torch.nn.functional.max_pool2d(y, 2, 2)
    return y.permute(0, 2, 3, 1).contiguous()


def cmd_beyond(a):
    import torch
    from oracle import quant
    dev = torch.device("cuda", 0)
    x, w, bd, wp, s_w, t_w = _layer(a, dev)
    xmax = float(x.abs().max())
    s_in, t_in = quant.activation_scales(xmax / 16.0)
    if a.fp16sat:
        s_in = quant.pow2_floor(2.0 ** 18 / xmax)          # max |x| s_in in [2^17, 2^18): fp16 saturates as well
    Ho, Wo = _out_hw(a)

    def run(s, t):
        inp, carried = _packed_input(x, s, t, dev)
        o32 = torch.full((a.B, Ho, Wo, a.cout), float("nan"), dtype=torch.float32, device=dev)
        _run(a, inp, wp, bd, a.flags | F_F32, 1.0 / (s * s_w), 1.0 / (2048.0 * t * t_w), 1.0, 1.0, o32)
        return o32, carried
    o32, (xh, xv, xr) = run(s_in, t_in)
    y = _ref64(a, x, w, bd, dev)                                       # true values
    a_ = argparse.Namespace(**{**vars(a), "flags": a.flags & F_POOL})
    mag = _ref64(a_, x.abs(), w.abs(), None, dev)                      # conv(|x|, |w|), max-pooled over the window
    scale = y.abs().max().item()
    err = (o32.double() - y).abs()
    cls = _quant_classes(x, s_in, t_in)
    finite = bool(torch.isfinite(o32).all())
    ratio = ((err - 2e-5 * scale).clamp_min(0) / mag.clamp_min(1e-30)).max().item()
    # the carried values, saturated e4m3 copies included, as gpu_checks.cmd_conv_f16f8 evaluates them: the kernel must use
    # what a saturated copy still holds (448 / t), not drop the cross terms of the saturated elements
    _, _, (wh, wv, wr) = quant.quantize(w.permute(2, 0, 1).contiguous(), s_w, t_w)
    wh, wv, wr = (z.permute(1, 2, 0).contiguous() for z in (wh, wv, wr))
    a0 = argparse.Namespace(**{**vars(a), "flags": 0})
    yc = _finish(a, _ref64(a0, xh, wh, None, dev) + _ref64(a0, xv, wr, None, dev) + _ref64(a0, xr, wv, None, dev), bd)
    carried_err = (o32.double() - yc).abs().max().item()
    # the same input calibrated on its true maximum (no saturation): the beyond-range error is measured against it
    o_cal, _ = run(*quant.activation_scales(xmax))
    cal_err = (o_cal.double() - y).abs().max().item()
    res = dict(s_in=s_in, t_in=t_in, classes=cls, finite=finite, max_err=err.max().item(), rel=err.max().item() / scale,
               scale=scale, err_over_conv_abs=ratio, gain=BEYOND_GAIN, carried_err=carried_err, calibrated_err=cal_err,
               over_calibrated=err.max().item() / max(cal_err, 1e-30))
    if a.fp16sat:
        ok = finite and cls["h_sat"] > 0
    else:
        ok = (finite and cls["v8_sat"] > 0 and cls["h_sat"] == 0 and carried_err <= 2e-5 * scale
              and bool((err <= BEYOND_GAIN * mag + 2e-5 * scale).all()))
    res["ok"] = bool(ok)
    print(json.dumps(res))
    return 0 if ok else 1


def cmd_net_scales(a):
    """Needs the test library (CTPN_B200_LIB=dbg)."""
    import ctypes as C
    import torch
    from ctpn_b200 import CtpnError, Engine
    from ctpn_b200 import _native as N
    from oracle import net_cpu, quant, synth
    names = [n for n, _, _, _ in net_cpu.CONV_LAYERS]                  # conv1_1 .. rpn_conv/3x3
    taps = [n + "+pool" if p else n for n, _, _, p in net_cpu.CONV_LAYERS[:13]]
    base = synth.make_weights(0)
    im = synth.make_image(a.seed, a.H, a.W)
    blob = (im.astype(np.float32) - net_cpu.PIXEL_MEANS.astype(np.float64)).astype(np.float32)[None]
    ref = net_cpu.forward(blob, base, dtype=torch.float64, taps=taps)
    ref_max = [float(np.abs(ref[t]).max()) for t in taps]
    eng = Engine(None, mode="f16f8", keep_activations=True)
    imd = torch.from_numpy(im[None]).cuda()
    res, ok = dict(cases=[]), True
    for layer, k in [(None, 0)] + [(l, e) for l, e in a.cases]:
        w = dict(base)
        c = 2.0 ** k
        if layer is not None:
            w[names[layer] + "/weights"] = base[names[layer] + "/weights"] * np.float32(c)
            w[names[layer] + "/biases"] = base[names[layer] + "/biases"] * np.float32(c)
            w[names[layer + 1] + "/weights"] = base[names[layer + 1] + "/weights"] * np.float32(1.0 / c)
        eng.load_weights(w)
        if k > 64:
            try:
                eng.forward_heads(imd)
                refused = ""
            except CtpnError as e:
                refused = str(e)
            good = "exceed 65504 * 2^48" in refused
            res["cases"].append(dict(layer=layer, k=k, refused=refused))
            ok = ok and good
            continue
        eng.forward_heads(imd)
        torch.cuda.synchronize()
        s, t, amax = ((C.c_float * 13)() for _ in range(3))
        N.check(N.lib.ctpn_net_f16f8_scales(eng._net, s, t, amax), "ctpn_net_f16f8_scales")
        s, t, amax = list(s), list(t), list(amax)
        want_max = [m * (c if l == layer else 1.0) for l, m in enumerate(ref_max)]
        bad_scales = [l for l in range(13) if (s[l], t[l]) != quant.activation_scales(amax[l])]
        # amax is read off the fp16 plane at the trial scale: fp16 rounding (2^-11) plus the arithmetic's own error
        bad_amax = [l for l in range(13) if abs(amax[l] - want_max[l]) > 2.0 ** -10 * want_max[l]]
        case = dict(layer=layer, k=k, s=s, t=t, amax=amax, bad_scales=bad_scales, bad_amax=bad_amax)
        good = not bad_scales and not bad_amax
        if layer is not None:
            # the scaled layer's debug tap decodes its planes at its own scale: c x the oracle's layer output
            got = eng.tap(taps[layer]).cpu().double().numpy()
            want = ref[taps[layer]].reshape(-1) * c
            case["tap_rel"] = float(np.abs(got - want).max() / np.abs(want).max())
            good = good and case["tap_rel"] < 5e-4
            if k >= 12:
                good = good and s[layer] < 1.0
        res["cases"].append(case)
        ok = ok and good
    res["ok"] = bool(ok)
    print(json.dumps(res))
    return 0 if ok else 1


def main(argv=None):
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    conv = dict(B=1, H=16, W=8, cin=64, cout=64, taps=9, flags=0, seed=0)
    specs = {"outq": conv, "sin": conv, "beyond": dict(conv, fp16sat=0), "conv1_eqv": dict(B=1, H=37, W=45, seed=0),
             "net_scales": dict(H=96, W=160, seed=7)}
    for name, defaults in specs.items():
        sp = sub.add_parser(name)
        for k, d in defaults.items():
            sp.add_argument("--" + k, type=int, default=d)
        if name in ("outq", "sin", "beyond"):
            sp.add_argument("--xscale", type=float, default=1.0)
    sub.choices["net_scales"].add_argument("--cases", type=lambda v: [tuple(int(z) for z in p.split(":")) for p in v.split(",")],
                                           default=[], help="layer:exponent,... (layer l and l + 1 rescaled by 2^k, 2^-k)")
    a = ap.parse_args(argv)
    fn = {"outq": cmd_outq, "sin": cmd_sin, "beyond": cmd_beyond, "conv1_eqv": cmd_conv1_eqv, "net_scales": cmd_net_scales}[a.cmd]
    rc, res = variant_checks._profiled(fn, a)
    print(json.dumps(res))
    return rc


if __name__ == "__main__":
    sys.exit(main())
