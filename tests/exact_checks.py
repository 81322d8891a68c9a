#!/usr/bin/env python
"""Stand-alone GPU checks of the convolutions in exact integer arithmetic (tests/exact_cases.py), run as subprocesses by
tests/test_exact_gpu.py so that a faulting kernel fails one test instead of the session.  Each sub-command prints one JSON
line {"ok": bool, "mismatches": n, "uncovered": n, "labels": [...], ...} as its last line of stdout; "labels" are the
conv_tc instantiations the profiler saw run (tests/variant_checks.py, parse_label).

The preconditions and the coverage of the case are evaluated in float64 first; a case that violates a precondition is
reported and never launched.  Then every output must equal the reference bit for bit:
    conv        ctpn_conv3x3 (--impl simt: ctpn_conv3x3_simt of the test library, every plane pair) -- bf16 planes and
                float32 outputs; with CTPN_F_STACK_IN the stacked output's image rows and zero pad rows, the compact planes
                and float32 outputs
    conv_f16f8  ctpn_conv3x3_f16f8 -- float32 output, F16F8 planes byte-identical to oracle.quant.quantize, and
                CTPN_F_OUT_BF16X2 planes
    conv1       ctpn_conv1_1_tc on a uint8 image + LUT (--blob 1: a float32 blob), planes 1 and 2
    conv1_q     ctpn_conv1_1_tc_f16f8, byte-identical to oracle.quant.quantize
    pack        ctpn_pack_weights against the plane split of the transposed TF layout, incl. cout_pad > cout

    python tests/exact_checks.py conv --B 1 --H 16 --W 8 --cin 64 --cout 64 --taps 9 --planes 3 --flags 3
    python tests/exact_checks.py conv_f16f8 --B 1 --H 9 --W 6 --cin 512 --cout 512 --taps 9 --flags 1

Several cases can share one process: separate their command lines with "+".  Each case then prints its own JSON line, and
the last line is {"ok", "mismatches", "uncovered", "cases": [the cases' results]}.

    python tests/exact_checks.py conv1 --planes 1 + conv1 --planes 2 --blob 1
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT, os.path.join(ROOT, "text-detection-ctpn_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import exact_cases as E  # noqa: E402


def compare(name, got, want, unit=1.0):
    """Bit-for-bit comparison of two tensors of one dtype; on a mismatch the count, first positions and got / want (floats
    in units of `unit`, bytes as integers)."""
    import torch
    assert got.shape == want.shape and got.dtype == want.dtype, (name, got.shape, want.shape, got.dtype, want.dtype)
    ib = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[got.element_size()]
    g, w = got.contiguous().view(ib), want.to(got.device).contiguous().view(ib)
    bad = g != w
    n = int(bad.sum().item())
    res = dict(mismatches=n)
    if n:
        idx = torch.nonzero(bad)[:8]
        conv = (lambda t: t.float().item() / unit) if got.dtype.is_floating_point else (lambda t: int(t.item()))
        res["first"] = idx.tolist()
        res["got"] = [conv(got[tuple(i)]) for i in idx.tolist()]
        res["want"] = [conv(want.to(got.device)[tuple(i)]) for i in idx.tolist()]
    return {name: res}


def _finish(res, runs, labels):
    """Prints the case's JSON line and returns it."""
    res["runs"] = runs
    res["mismatches"] = sum(r["mismatches"] for r in runs.values())
    res["labels"] = labels
    res["ok"] = bool(not res.get("violated") and res["mismatches"] == 0 and res["uncovered"] == 0)
    print(json.dumps(res))
    return res


def _pre(case, ops, pairs="tc"):
    bounds, bad = E.check_preconditions(case, ops, pairs)
    miss, ntiles = E.coverage(case, ops, pairs)
    res = dict(bounds=bounds, tiles=ntiles, uncovered=sum(miss.values()),
               uncovered_terms={k: v for k, v in miss.items() if v})
    if bad:
        res["violated"] = bad
    return res


def _prof(on):
    from ctpn_b200 import _native as N
    N.check(N.lib.ctpn_prof_enable(1 if on else 0), "ctpn_prof_enable")


def _labels():
    from variant_checks import conv_tc_labels
    return conv_tc_labels()


def cmd_conv(a):
    import torch
    from ctpn_b200 import _native as N
    dev = torch.device("cuda", 0)
    case = E.conv(a.B, a.H, a.W, a.cin, a.cout, a.taps, a.planes, a.flags)
    pairs = "all" if a.impl == "simt" else "tc"
    ops = {k: v.to(dev) for k, v in E.bf16_operands(case, a.seed).items()}
    res = _pre(case, ops, pairs)
    if res.get("violated"):
        return _finish(res, {}, [])
    y32 = E.reference(case, ops, pairs).float()                 # exact
    P, B, Co = a.planes, a.B, a.cout
    Ho, Wo = y32.shape[1], y32.shape[2]
    xin, wp = E.bf16_inputs(ops)
    bias = ops["bias"].float().contiguous()
    fn = N.lib.ctpn_conv3x3_simt if a.impl == "simt" else N.lib.ctpn_conv3x3
    stack_in = bool(a.flags & E.F_STACK_IN)
    if stack_in:
        xin = E.stacked(xin).contiguous()

    def run(flags):
        rows = Ho + 1 if flags & E.F_STACK_OUT else Ho
        if flags & E.F_F32:
            out = torch.full((B, rows, Wo, Co), float("nan"), dtype=torch.float32, device=dev)
        else:
            out = torch.full((P, B, rows, Wo, Co), float("nan"), dtype=torch.bfloat16, device=dev)
        N.check(fn(N.ptr(xin), N.ptr(wp), N.ptr(bias), N.ptr(out), B, a.H, a.W, a.cin, Co, a.taps, P, flags, N.stream_ptr()),
                "conv")
        torch.cuda.synchronize()
        return out
    want_p = E.split_planes(y32, P)
    base = a.flags & ~(E.F_F32 | E.F_STACK_OUT)
    runs = {}
    _prof(True)
    if a.flags & E.F_STACK_OUT:
        so = run(base | E.F_STACK_OUT)
        runs.update(compare("stacked_planes", so[:, :, :Ho], want_p))
        runs.update(compare("stacked_pad_rows", so[:, :, Ho], torch.zeros_like(so[:, :, Ho])))
    runs.update(compare("planes", run(base), want_p))
    runs.update(compare("f32", run(base | E.F_F32), y32))
    labels = _labels()
    _prof(False)
    res["stacked_in"] = stack_in
    return _finish(res, runs, labels)


def cmd_conv_f16f8(a):
    import torch
    from ctpn_b200 import _native as N
    from oracle import quant
    dev = torch.device("cuda", 0)
    case = E.f16f8(a.B, a.H, a.W, a.cin, a.cout, a.taps, a.flags, a.cross_fill)
    ops = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in E.f16f8_operands(case, a.seed).items()}
    res = _pre(case, ops)
    if res.get("violated"):
        return _finish(res, {}, [])
    y32 = E.reference(case, ops).float()
    B, Co = a.B, a.cout
    Ho, Wo = y32.shape[1], y32.shape[2]
    act, wt = (t.to(dev) for t in E.f16f8_inputs(ops))
    bias = ops["bias"].float().contiguous()
    amax = max(float(y32.abs().max()), 1.0)
    out_s = 2.0 if amax * 2.0 <= 16384.0 else 1.0                # exercise the fp16 pre-scale where it fits
    out_t = quant.pow2_floor(448.0 / amax) / 2.0
    res.update(out_s=out_s, out_t=out_t, inv_main=ops["inv_main"], inv_cross=ops["inv_cross"])

    def run(flags, out):
        N.check(N.lib.ctpn_conv3x3_f16f8(N.ptr(act), N.ptr(wt), N.ptr(bias), N.ptr(out), B, a.H, a.W, a.cin, Co, a.taps, flags,
                                         ops["inv_main"], ops["inv_cross"], out_s, out_t, N.stream_ptr()), "conv_f16f8")
        torch.cuda.synchronize()
        return out
    base = a.flags & ~(E.F_F32 | E.F_OUT_BF16X2)
    nel = B * Ho * Wo * Co
    runs = {}
    _prof(True)
    o32 = run(base | E.F_F32, torch.full((B, Ho, Wo, Co), float("nan"), dtype=torch.float32, device=dev))
    runs.update(compare("f32", o32, y32, unit=min(ops["inv_main"], ops["inv_cross"])))
    oq = run(base, torch.full((nel * 4,), 0xFF, dtype=torch.uint8, device=dev))
    h, cross, _ = quant.quantize(y32.cpu(), out_s, out_t)
    runs.update(compare("f16f8_fp16_plane", oq[:nel * 2], h.contiguous().view(torch.uint8).reshape(-1)))
    runs.update(compare("f16f8_e4m3_plane", oq[nel * 2:], cross.reshape(-1)))
    ob = run(base | E.F_OUT_BF16X2, torch.full((2, B, Ho, Wo, Co), float("nan"), dtype=torch.bfloat16, device=dev))
    runs.update(compare("bf16x2", ob, E.split_planes(y32, 2)))
    labels = _labels()
    _prof(False)
    return _finish(res, runs, labels)


def _conv1(a, outq):
    import torch
    from ctpn_b200 import _native as N
    from oracle import quant
    dev = torch.device("cuda", 0)
    P = 2 if outq else a.planes
    ops = E.conv1_operands(a.B, a.H, a.W, a.seed, blob=bool(a.blob))
    bounds, bad, miss, ntiles, y = E.conv1_check(ops, P)
    res = dict(bounds=bounds, tiles=ntiles, uncovered=sum(miss.values()), uncovered_terms={k: v for k, v in miss.items() if v})
    if bad:
        res["violated"] = bad
        return _finish(res, {}, [])
    y32 = y.clamp_min(0.0).float()
    w = ops["w"].float().to(dev).contiguous()
    bias = ops["bias"].float().to(dev).contiguous()
    if a.blob:
        src, lut = ops["x"].float().to(dev).contiguous(), None
    else:
        src, lut = ops["im"].to(dev).contiguous(), ops["lut"].float().to(dev).contiguous()
    nel = a.B * a.H * a.W * 64
    runs = {}
    _prof(True)
    if outq:
        amax = max(float(y32.abs().max()), 1.0)
        out_s, out_t = quant.pow2_floor(16384.0 / amax), quant.pow2_floor(448.0 / amax) / 2.0
        out = torch.full((nel * 4,), 0xFF, dtype=torch.uint8, device=dev)
        N.check(N.lib.ctpn_conv1_1_tc_f16f8(N.ptr(src), a.blob, N.ptr(lut), N.ptr(w), N.ptr(bias), N.ptr(out), a.B, a.H, a.W,
                                            out_s, out_t, N.stream_ptr()), "conv1_1_tc_f16f8")
        torch.cuda.synchronize()
        h, cross, _ = quant.quantize(y32, out_s, out_t)
        runs.update(compare("f16f8_fp16_plane", out[:nel * 2], h.contiguous().view(torch.uint8).reshape(-1)))
        runs.update(compare("f16f8_e4m3_plane", out[nel * 2:], cross.reshape(-1)))
        res.update(out_s=out_s, out_t=out_t)
    else:
        out = torch.full((P, a.B, a.H, a.W, 64), float("nan"), dtype=torch.bfloat16, device=dev)
        N.check(N.lib.ctpn_conv1_1_tc(N.ptr(src), a.blob, N.ptr(lut), N.ptr(w), N.ptr(bias), N.ptr(out), a.B, a.H, a.W, P,
                                      N.stream_ptr()), "conv1_1_tc")
        torch.cuda.synchronize()
        runs.update(compare("planes", out, E.split_planes(y32, P)))
    labels = _labels()
    _prof(False)
    return _finish(res, runs, labels)


def cmd_conv1(a):
    return _conv1(a, False)


def cmd_conv1_q(a):
    return _conv1(a, True)


PACK_SHAPES = [   # (taps, cin, cout, cout_pad, planes)
    (9, 64, 64, 64, 1), (9, 128, 96, 128, 2), (9, 512, 512, 512, 3), (1, 512, 20, 64, 3), (1, 256, 1000, 1024, 2),
]


def cmd_pack(a):
    """ctpn_pack_weights bit for bit: planes [P][cout_pad][taps][Cin] = the plane split of w_tf transposed to
    [Cout][taps][Cin], zero rows for cout <= co < cout_pad.  Weights: float32 normals over several binades (all 24 bits
    set, so the third plane is not zero) and exact zeros."""
    import torch
    from ctpn_b200 import _native as N
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(a.seed)
    runs = {}
    for taps, cin, cout, cout_pad, P in PACK_SHAPES:
        w = torch.randn(taps, cin, cout, generator=g) * torch.exp2(torch.randint(-12, 6, (taps, cin, cout), generator=g).float())
        w[torch.rand(taps, cin, cout, generator=g) < 0.05] = 0.0
        want = torch.zeros((P, cout_pad, taps, cin), dtype=torch.bfloat16)
        want[:, :cout] = E.split_planes(w.permute(2, 0, 1).contiguous(), P)
        out = torch.full((P * cout_pad * taps * cin,), float("nan"), dtype=torch.bfloat16, device=dev)
        wd = w.to(dev).contiguous()
        N.check(N.lib.ctpn_pack_weights(N.ptr(wd), taps, cin, cout, cout_pad, P, N.ptr(out), N.stream_ptr()), "pack")
        torch.cuda.synchronize()
        runs.update(compare("t%d_c%d-%d_pad%d_p%d" % (taps, cin, cout, cout_pad, P), out.view(want.shape), want))
    return _finish(dict(uncovered=0), runs, [])


def run_case(argv):
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    specs = {
        "conv": dict(B=1, H=8, W=16, cin=64, cout=64, taps=9, planes=1, flags=0, seed=0),
        "conv_f16f8": dict(B=1, H=8, W=16, cin=64, cout=64, taps=9, flags=0, seed=0),
        "conv1": dict(B=1, H=37, W=45, planes=2, blob=0, seed=0),
        "conv1_q": dict(B=1, H=37, W=45, blob=0, seed=0),
        "pack": dict(seed=0),
    }
    for name, defaults in specs.items():
        sp = sub.add_parser(name)
        for k, d in defaults.items():
            sp.add_argument("--" + k, type=int, default=d)
    sub.choices["conv"].add_argument("--impl", default="tc", choices=["tc", "simt"])
    sub.choices["conv_f16f8"].add_argument("--cross_fill", type=float, default=None)
    a = ap.parse_args(argv)
    fn = {"conv": cmd_conv, "conv_f16f8": cmd_conv_f16f8, "conv1": cmd_conv1, "conv1_q": cmd_conv1_q, "pack": cmd_pack}[a.cmd]
    try:
        res = fn(a)
    finally:
        try:
            _prof(False)
        except Exception:
            pass
    res["case"] = " ".join(argv)
    return res


def main(argv=None):
    argv = sys.argv[1:] if argv is None else argv
    cases, cur = [], []
    for tok in argv + ["+"]:
        if tok == "+":
            if cur:
                cases.append(cur)
            cur = []
        else:
            cur.append(tok)
    results = [run_case(c) for c in cases]
    if len(results) > 1:
        res = dict(ok=all(r["ok"] for r in results), mismatches=sum(r["mismatches"] for r in results),
                   uncovered=sum(r["uncovered"] for r in results), cases=results)
        print(json.dumps(res))
    return 0 if all(r["ok"] for r in results) else 1


if __name__ == "__main__":
    sys.exit(main())
