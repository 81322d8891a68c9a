#!/usr/bin/env python
"""Stand-alone GPU checks that also report which conv_tc instantiation ran, run as subprocesses by
tests/test_kernel_variants_gpu.py so that a faulting kernel fails one test instead of the session.  Each sub-command prints
one JSON line {"ok": bool, "labels": [...], ...} as its last line of stdout.

conv, conv_f16f8 and conv1 run the command of the same name in tests/gpu_checks.py with launch profiling on, and add the
profiler's "conv_tc ..." kernel labels to its result; a label names the template instantiation that ran
(csrc/conv_tc.cu, launch_bn), see parse_label.  The other sub-commands are checks gpu_checks.py does not have:

    conv1_q       ctpn_conv1_1_tc_f16f8 (conv1_1 writing F16F8 planes) against float64
    conv1_f32     ctpn_conv1_1_tc on a float32 blob (src_is_f32 = 1) against float64
    stack_planes  CTPN_F_STACK_IN / _OUT of ctpn_conv3x3 on bf16 planes, bit for bit against the plain layout

    python tests/variant_checks.py conv --B 1 --H 16 --W 8 --cin 64 --cout 64 --taps 9 --planes 3 --flags 3
    python tests/variant_checks.py stack_planes --B 3 --H 13 --W 8 --cin 64 --cout 64 --planes 3 --promote 1
"""
import argparse
import contextlib
import io
import json
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT, os.path.join(ROOT, "text-detection-ctpn_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import gpu_checks  # noqa: E402
from gpu_checks import F_POOL, F_RELU  # noqa: E402

F_F32, F_STACK_IN, F_STACK_OUT, F_PROMOTE = 4, 16, 32, 64
# bounds of gpu_checks.cmd_conv (bf16 plane output) and cmd_conv1 (tensor-core kernel), per plane count
CONV_TOL = {1: 6e-3, 2: 4e-5, 3: 2e-5}
CONV1_TOL = {1: 1.2e-2, 2: 6e-5, 3: 3e-6}

_LABEL = re.compile(r"^conv_tc t(\d+) (\d+)x(\d+)x(\d+) c(\d+)-(\d+) (f16f8 )?p(\d) bn(\d+)( mc)?( promote)?$")


def parse_label(label):
    """'conv_tc t9 1x37x56 c512-512 p3 bn128 mc promote' -> (taps, f16f8, planes, BN, mc, promote) = (9, 0, 3, 128, 1, 1)."""
    m = _LABEL.match(label)
    if m is None:
        raise ValueError("not a conv_tc kernel label: %r" % label)
    return (int(m.group(1)), int(bool(m.group(7))), int(m.group(8)), int(m.group(9)), int(bool(m.group(10))),
            int(bool(m.group(11))))


def conv_tc_labels():
    """Kernel labels of every conv_tc launch recorded since ctpn_prof_enable(1), sorted."""
    from ctpn_b200 import _native as N
    return sorted({r["kernel"] for r in N.prof_report() if r["kernel"].startswith("conv_tc ")})


def _profiled(fn, a):
    """Runs a gpu_checks command with profiling on and its stdout captured; returns (exit code, its result + labels)."""
    from ctpn_b200 import _native as N
    N.check(N.lib.ctpn_prof_enable(1), "ctpn_prof_enable")
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        rc = fn(a)
    lines = [l for l in buf.getvalue().splitlines() if l.startswith("{")]
    res = json.loads(lines[-1]) if lines else dict(ok=False, error="no result line", stdout=buf.getvalue()[-2000:])
    res["labels"] = conv_tc_labels()
    N.check(N.lib.ctpn_prof_enable(0), "ctpn_prof_enable")
    return rc, res


def _conv1_weights(rs):
    """conv1_1 weights, bias and mean-subtraction LUT drawn as gpu_checks.cmd_conv1 draws them."""
    w = (rs.standard_normal((3, 3, 3, 64)) * (2.0 / 27) ** 0.5 / 75.0).astype(np.float32)
    b = (rs.standard_normal(64) * 0.1).astype(np.float32)
    means = np.array([102.9801, 115.9465, 122.7717])
    lut = (np.arange(256, dtype=np.float64)[:, None] - means[None, :]).astype(np.float32)
    return w, b, lut


def _conv1_ref(x64, w, bd):
    """float64 conv1_1 (3x3 SAME, bias, ReLU) of an NHWC float64 device tensor -> NHWC."""
    import torch
    wr = torch.from_numpy(w.astype(np.float64)).to(x64.device).permute(3, 2, 0, 1)
    return torch.relu(torch.nn.functional.conv2d(x64.permute(0, 3, 1, 2), wr, bd.double(), padding=1)).permute(0, 2, 3, 1)


def cmd_conv1_q(a):
    """ctpn_conv1_1_tc_f16f8 on a uint8 image: the F16F8 planes decoded as gpu_checks.cmd_conv_f16f8 decodes them.
    fp16 value + residual within 6e-5 of max|y|, the e4m3 copy within 0.07 relative (with a subnormal floor)."""
    import torch
    from ctpn_b200 import _native as N
    dev = torch.device("cuda", 0)
    rs = np.random.RandomState(a.seed)
    im = rs.randint(0, 256, size=(a.B, a.H, a.W, 3)).astype(np.uint8)
    w, b, lut = _conv1_weights(rs)
    imd, wd, bd, lutd = (torch.from_numpy(x).to(dev) for x in (im, w, b, lut))
    x = torch.from_numpy(lut.astype(np.float64)[im.reshape(-1, 3), np.arange(3)].reshape(im.shape)).to(dev)
    y = _conv1_ref(x, w, bd)
    scale = y.abs().max().item()
    out_s, out_t = 1.0, gpu_checks._pow2_floor(448.0 / max(scale, 1e-6)) / 2.0
    nel = a.B * a.H * a.W * 64
    oq = torch.zeros(nel * 4, dtype=torch.uint8, device=dev)
    N.check(N.lib.ctpn_conv1_1_tc_f16f8(N.ptr(imd), 0, N.ptr(lutd), N.ptr(wd), N.ptr(bd), N.ptr(oq), a.B, a.H, a.W, out_s, out_t,
                                        N.stream_ptr()), "conv1_1_tc_f16f8")
    torch.cuda.synchronize()
    h = oq[:nel * 2].view(torch.float16).double().view(a.B, a.H, a.W, 64)
    cr = oq[nel * 2:].view(a.B, a.H, a.W, 128)
    v8 = cr[..., :64].contiguous().view(torch.float8_e4m3fn).double() / out_t
    r8 = cr[..., 64:].contiguous().view(torch.float8_e4m3fn).double() / (2048.0 * out_t)
    finite = bool(torch.isfinite(h).all().item() and torch.isfinite(v8).all().item() and torch.isfinite(r8).all().item())
    eq_hr = ((h / out_s + r8) - y).abs().max().item()
    eq_v8 = ((v8 - y).abs() / (y.abs() + scale * 2.0 ** -9)).max().item()
    ok = finite and eq_hr <= 6e-5 * scale and eq_v8 <= 0.07
    print(json.dumps(dict(ok=bool(ok), scale=scale, q_err_h_plus_r=eq_hr, rel=eq_hr / max(scale, 1e-30), q_rel_err_e4m3=eq_v8)))
    return 0 if ok else 1


def cmd_conv1_f32(a):
    """ctpn_conv1_1_tc with src_is_f32 = 1: a float32 blob with non-integer values (as _get_image_blob makes them after a
    rescale), no LUT; the bounds of gpu_checks.cmd_conv1."""
    import torch
    from ctpn_b200 import _native as N
    dev = torch.device("cuda", 0)
    rs = np.random.RandomState(a.seed)
    blob = rs.uniform(-130.0, 155.0, size=(a.B, a.H, a.W, 3)).astype(np.float32)
    w, b, _ = _conv1_weights(rs)
    xd, wd, bd = (torch.from_numpy(x).to(dev) for x in (blob, w, b))
    out = torch.zeros((a.planes, a.B, a.H, a.W, 64), dtype=torch.bfloat16, device=dev)
    N.check(N.lib.ctpn_conv1_1_tc(N.ptr(xd), 1, None, N.ptr(wd), N.ptr(bd), N.ptr(out), a.B, a.H, a.W, a.planes, N.stream_ptr()),
            "conv1_1_tc")
    torch.cuda.synchronize()
    got = out.double().sum(0)
    y = _conv1_ref(xd.double(), w, bd)
    err = (got - y).abs().max().item()
    scale = y.abs().max().item()
    tol = CONV1_TOL[a.planes]
    ok = bool(torch.isfinite(got).all().item()) and err <= tol * scale
    print(json.dumps(dict(ok=bool(ok), max_err=err, scale=scale, rel=err / max(scale, 1e-30), tol=tol)))
    return 0 if ok else 1


def cmd_stack_planes(a):
    """Row-stacked batches on bf16 planes: the checks of gpu_checks.cmd_conv_stack for ctpn_conv3x3.  Stacked input with
    stacked output (image rows equal the plain layout, pad rows zero), stacked input with compact plane and float32 outputs
    (equal the plain layout), and a pooled layer with a plain input writing a stacked output (image rows equal the plain
    pooled output, pad rows untouched).  The plain run itself is held to float64 on the first and last image."""
    import torch
    from ctpn_b200 import _native as N
    dev = torch.device("cuda", 0)
    g = torch.Generator(device="cpu").manual_seed(a.seed)
    B, H, W, C, Co, P = a.B, a.H, a.W, a.cin, a.cout, a.planes
    x = torch.relu(torch.randn(B, H, W, C, generator=g))
    w = torch.randn(9, C, Co, generator=g) * (2.0 / (9 * C)) ** 0.5
    b = torch.randn(Co, generator=g) * 0.1
    plain = gpu_checks.split_planes_t(x.to(dev), P).contiguous()                   # [P][B][H][W][C]
    stacked = torch.zeros((P, B, H + 1, W, C), dtype=torch.bfloat16, device=dev)     # one zero row after every image
    stacked[:, :, :H] = plain
    wp = torch.empty(P * Co * 9 * C, dtype=torch.bfloat16, device=dev)
    N.check(N.lib.ctpn_pack_weights(N.ptr(w.to(dev).contiguous()), 9, C, Co, Co, P, N.ptr(wp), N.stream_ptr()), "pack")
    bd = b.to(dev)
    extra = F_PROMOTE if a.promote else 0

    def run(inp, flags, nbytes):
        out = torch.full((nbytes,), 0xAB, dtype=torch.uint8, device=dev)
        N.check(N.lib.ctpn_conv3x3(N.ptr(inp), N.ptr(wp), N.ptr(bd), N.ptr(out), B, H, W, C, Co, 9, P, flags | extra,
                                   N.stream_ptr()), "conv")
        torch.cuda.synchronize()
        return out
    n, ns = B * H * W * Co, B * (H + 1) * W * Co                  # elements per plane, compact / stacked
    ref = run(plain, F_RELU, P * 2 * n)                           # plain in, plain out
    so = run(stacked, F_RELU | F_STACK_IN | F_STACK_OUT, P * 2 * ns)
    co = run(stacked, F_RELU | F_STACK_IN, P * 2 * n)             # stacked in, compact planes out
    cf = run(stacked, F_RELU | F_STACK_IN | F_F32, 4 * n)         # stacked in, compact float32 out
    rf = run(plain, F_RELU | F_F32, 4 * n)
    ok_compact = bool(torch.equal(co, ref)) and bool(torch.equal(cf, rf))
    r4, s4 = ref.view(P, B, H, -1), so.view(P, B, H + 1, -1)
    ok_rows = bool(torch.equal(s4[:, :, :H], r4))
    ok_pad = bool((s4[:, :, H] == 0).all())
    Hp, Wp = H // 2, W // 2
    n2, n2s = B * Hp * Wp * Co, B * (Hp + 1) * Wp * Co
    pp = run(plain, F_RELU | F_POOL, P * 2 * n2).view(P, B, Hp, -1)
    ps = run(plain, F_RELU | F_POOL | F_STACK_OUT, P * 2 * n2s).view(P, B, Hp + 1, -1)
    ok_pool = bool(torch.equal(ps[:, :, :Hp], pp)) and bool((ps[:, :, Hp] == 0xAB).all())
    # the plain run against float64 on the values the planes carry (first and last image: the stack's ends)
    sel = [0, B - 1] if B > 1 else [0]
    xr = plain.double().sum(0)[sel].permute(0, 3, 1, 2)
    wr = wp.view(P, Co, 9, C).double().sum(0).view(Co, 3, 3, C).permute(0, 3, 1, 2)
    y = torch.relu(torch.nn.functional.conv2d(xr, wr, bd.double(), padding=1)).permute(0, 2, 3, 1)
    got = ref.view(torch.bfloat16).view(P, B, H, W, Co).double().sum(0)[sel]
    scale = y.abs().max().item()
    max_err = (got - y).abs().max().item()
    ok_f64 = max_err <= CONV_TOL[P] * max(scale, 1e-6)
    ok = ok_compact and ok_rows and ok_pad and ok_pool and ok_f64
    print(json.dumps(dict(ok=bool(ok), compact=ok_compact, rows=ok_rows, pad_zero=ok_pad, pooled_stack_out=ok_pool, f64=bool(ok_f64),
                          max_err=max_err, scale=scale, tol=CONV_TOL[P])))
    return 0 if ok else 1


def main(argv=None):
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    specs = {
        "conv": dict(B=1, H=8, W=16, cin=64, cout=64, taps=9, planes=1, flags=0, seed=0, nonneg=0),
        "conv_f16f8": dict(B=1, H=8, W=16, cin=64, cout=64, taps=9, flags=0, seed=0),
        "conv1": dict(B=1, H=37, W=45, planes=2, seed=0),
        "conv1_q": dict(B=1, H=37, W=45, seed=0),
        "conv1_f32": dict(B=1, H=37, W=45, planes=2, seed=0),
        "stack_planes": dict(B=3, H=37, W=56, cin=128, cout=128, planes=2, promote=0, seed=0),
    }
    for name, defaults in specs.items():
        sp = sub.add_parser(name)
        for k, d in defaults.items():
            sp.add_argument("--" + k, type=int, default=d)
    sub.choices["conv"].add_argument("--impl", default="tc")
    sub.choices["conv1"].add_argument("--impl", default="tc")
    sub.choices["conv_f16f8"].add_argument("--xscale", type=float, default=1.0)
    a = ap.parse_args(argv)
    fn = {"conv": gpu_checks.cmd_conv, "conv_f16f8": gpu_checks.cmd_conv_f16f8, "conv1": gpu_checks.cmd_conv1,
          "conv1_q": cmd_conv1_q, "conv1_f32": cmd_conv1_f32, "stack_planes": cmd_stack_planes}[a.cmd]
    rc, res = _profiled(fn, a)
    print(json.dumps(res))
    return rc


if __name__ == "__main__":
    sys.exit(main())
