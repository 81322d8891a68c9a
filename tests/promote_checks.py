#!/usr/bin/env python
"""Stand-alone GPU check of CTPN_F_PROMOTE, run as a subprocess by tests/test_promote_gpu.py so that a faulting kernel
cannot poison the pytest process.  Prints one JSON line {"ok": bool, ...} as its last line of stdout.

ctpn_conv3x3 on three bf16 planes runs with and without the flag on the same inputs, and both results are compared with a
float64 conv2d on the exact operand values the planes carry.  It reports max |error| and mean signed error of both runs;
--nonneg 1 makes every product positive (non-negative activations and weights), so the tensor core's truncation shows as
a negative mean.

    python tests/promote_checks.py --B 1 --H 37 --W 56 --cin 512 --cout 512 --taps 9 --flags 5 --nonneg 1
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "text-detection-ctpn_b200"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

F_RELU, F_POOL, F_F32, F_PROMOTE = 1, 2, 4, 64


def main(argv=None):
    ap = argparse.ArgumentParser()
    for k, d in dict(B=1, H=37, W=56, cin=512, cout=512, taps=9, flags=1, seed=0, nonneg=0).items():
        ap.add_argument("--" + k, type=int, default=d)
    a = ap.parse_args(argv)
    import torch
    from ctpn_b200 import _native as N
    from gpu_checks import split_planes_t
    dev = torch.device("cuda", 0)
    g = torch.Generator(device="cpu").manual_seed(a.seed)
    x = torch.randn(a.B, a.H, a.W, a.cin, generator=g)
    w = torch.randn(a.taps, a.cin, a.cout, generator=g) * (2.0 / (a.taps * a.cin)) ** 0.5
    b = torch.randn(a.cout, generator=g) * 0.1
    if a.nonneg:
        x, w, b = torch.relu(x), w.abs(), b.abs()
    xp = split_planes_t(x.to(dev), 3).contiguous()
    wp = torch.empty(3 * a.cout * a.taps * a.cin, dtype=torch.bfloat16, device=dev)
    w_dev, b_dev = w.to(dev).contiguous(), b.to(dev).contiguous()
    N.check(N.lib.ctpn_pack_weights(N.ptr(w_dev), a.taps, a.cin, a.cout, a.cout, 3, N.ptr(wp), N.stream_ptr()), "pack")
    k = 3 if a.taps == 9 else 1
    wr = wp.view(3, a.cout, a.taps, a.cin).double().sum(0).view(a.cout, k, k, a.cin).permute(0, 3, 1, 2)
    y = torch.nn.functional.conv2d(xp.double().sum(0).permute(0, 3, 1, 2), wr, b_dev.double(), padding=k // 2)
    if a.flags & F_RELU:
        y = torch.relu(y)
    if a.flags & F_POOL:
        y = torch.nn.functional.max_pool2d(y, 2, 2)
    y = y.permute(0, 2, 3, 1)
    Ho, Wo = y.shape[1], y.shape[2]
    scale = y.abs().max().item()
    res = dict(scale=scale, K=a.taps * a.cin)
    for tag, flags in (("plain", a.flags), ("promoted", a.flags | F_PROMOTE)):
        if a.flags & F_F32:
            out = torch.full((a.B, Ho, Wo, a.cout), float("nan"), dtype=torch.float32, device=dev)
        else:
            out = torch.zeros((3, a.B, Ho, Wo, a.cout), dtype=torch.bfloat16, device=dev)
        N.check(N.lib.ctpn_conv3x3(N.ptr(xp), N.ptr(wp), N.ptr(b_dev), N.ptr(out), a.B, a.H, a.W, a.cin, a.cout, a.taps, 3,
                                   flags, N.stream_ptr()), "conv")
        torch.cuda.synchronize()
        got = out.double() if a.flags & F_F32 else out.double().sum(0)
        d = got - y
        res[tag] = dict(max_err=d.abs().max().item(), mean_err=d.mean().item(), nan=int(torch.isnan(got).sum().item()))
    # both runs stay inside the bf16x3 bound of the plain kernel checks (2e-5 of max |y|); the tests compare the two errors
    ok = all(res[t]["nan"] == 0 and res[t]["max_err"] <= 2e-5 * max(scale, 1e-6) for t in ("plain", "promoted"))
    res["ok"] = bool(ok)
    print(json.dumps(res))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
