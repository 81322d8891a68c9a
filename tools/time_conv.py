#!/usr/bin/env python
"""Perf experiment (test library: honours CTPN_TC_BN / CTPN_TC_STAGES_A / CTPN_TC_STAGES_B / CTPN_TC_MCAST / CTPN_TC_DEBUG /
CTPN_TC_PROMOTE): time one 3x3 layer of the conv stack alone, bf16 planes, bf16x3 with promoted accumulation, or F16F8.

    CTPN_TC_STAGES_B=2 python tools/time_conv.py --B 32 --H 75 --W 112 --cin 512 --cout 512 --mode f16f8
    CTPN_TC_PROMOTE=4 python tools/time_conv.py --B 32 --H 37 --W 56 --cin 512 --cout 512 --mode bf16x3p
"""
import argparse
import os
import sys

os.environ.setdefault("CTPN_B200_LIB", "dbg")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "text-detection-ctpn_b200"))
import torch  # noqa: E402
from ctpn_b200 import _native as N  # noqa: E402

ap = argparse.ArgumentParser()
for k, d in dict(B=32, H=75, W=112, cin=512, cout=512, flags=1, reps=20).items():
    ap.add_argument("--" + k, type=int, default=d)
ap.add_argument("--mode", default="f16f8")
a = ap.parse_args()
dev = torch.device("cuda", 0)
planes = {"bf16": 1, "bf16x2": 2, "bf16x3": 3, "bf16x3p": 3, "f16f8": 2}[a.mode]
flags = a.flags | (64 if a.mode == "bf16x3p" else 0)       # CTPN_F_PROMOTE (interval: CTPN_TC_PROMOTE)
nin = a.B * a.H * a.W * a.cin
x = torch.randint(0, 60, (planes * nin * 2,), dtype=torch.uint8, device=dev)            # small positive operand bytes
w = torch.randint(0, 60, (planes * a.cout * 9 * a.cin * 2,), dtype=torch.uint8, device=dev)
b = torch.zeros(a.cout, dtype=torch.float32, device=dev)
pool = bool(a.flags & 2)
Ho, Wo = (a.H // 2, a.W // 2) if pool else (a.H, a.W)
out = torch.empty(planes * a.B * Ho * Wo * a.cout * 2, dtype=torch.uint8, device=dev)


def run():
    if a.mode == "f16f8":
        N.check(N.lib.ctpn_conv3x3_f16f8(N.ptr(x), N.ptr(w), N.ptr(b), N.ptr(out), a.B, a.H, a.W, a.cin, a.cout, 9, a.flags, 1.0, 1.0, 1.0, 1.0, N.stream_ptr()), "conv")
    else:
        N.check(N.lib.ctpn_conv3x3(N.ptr(x), N.ptr(w), N.ptr(b), N.ptr(out), a.B, a.H, a.W, a.cin, a.cout, 9, planes, flags, N.stream_ptr()), "conv")


for _ in range(3):
    run()
torch.cuda.synchronize()
ts = []
for _ in range(a.reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); run(); e1.record(); torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
ts.sort()
fl = 2.0 * a.B * a.H * a.W * 9 * a.cin * a.cout
env = " ".join("%s=%s" % (k, v) for k, v in sorted(os.environ.items()) if k.startswith("CTPN_TC"))
print("%s %dx%dx%d c%d-%d f%d [%s]: median %.3f ms (min %.3f)  %.0f alg TFLOP/s" % (a.mode, a.B, a.H, a.W, a.cin, a.cout, a.flags, env, ts[len(ts) // 2], ts[0], fl / ts[len(ts) // 2] / 1e9), flush=True)
