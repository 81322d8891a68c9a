#!/usr/bin/env python
"""Where the time of the flagship's 3x3 layers goes (test library, CTPN_B200_LIB=dbg): each of the thirteen conv_tc 3x3
launches of batch 32 x 600x900 timed alone with CUDA events, plain and with one part of the pipeline switched off or
re-sized.

    python tools/conv_pipeline.py > profiles/conv_epilogue_before.txt
    python tools/conv_pipeline.py --cols plain,-B,-A --stages-b 2,3,4,6

Columns (one child process per column, since the library reads the CTPN_TC_* switches once):
    plain        the product configuration
    -B / -A      CTPN_TC_DEBUG=1 / 2: weight / activation TMA loads skipped (the barriers still flip)
    -MMA         CTPN_TC_DEBUG=4: the wgmma instructions skipped
    -epi         CTPN_TC_DEBUG=16: the epilogue's staging, arithmetic and stores skipped
    -epi-st      CTPN_TC_DEBUG=24: -epi and the stores
    sb=N         CTPN_TC_STAGES_B=N: at most N weight stages (the layout's own count when it has fewer: 3 at BN = 128,
                 6 at BN = 64 for both modes)
Each cell is the median of --reps launches after three warm-up launches, in ms.  'floor' is the layer's MMA time at the
H100 SXM data-sheet rate (989 dense bf16 TFLOP/s) in the mode's bf16-rate MMA units per MAC (f16f8 2, bf16x2 3).  The
'sum' row is the conv_tc 3x3 time of one flagship step.  The card's name, power limit and SM clock (read by each child
right after its last launch) are printed with the table.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RELU, POOL, OUT_BF16X2, STACK_IN, STACK_OUT = 1, 2, 8, 16, 32
# name, B, H, W, Cin, Cout, flags: the flagship's conv_tc 3x3 launches at batch 32 x 600x900 (ctpn_net_forward's layer
# list; conv4_3's pooled output and the 1/16-scale maps are row-stacked)
SHAPES = [
    ("conv1_2", 32, 600, 900, 64, 64, RELU | POOL),
    ("conv2_1", 32, 300, 450, 64, 128, RELU),
    ("conv2_2", 32, 300, 450, 128, 128, RELU | POOL),
    ("conv3_1", 32, 150, 225, 128, 256, RELU),
    ("conv3_2", 32, 150, 225, 256, 256, RELU),
    ("conv3_3", 32, 150, 225, 256, 256, RELU | POOL),
    ("conv4_1", 32, 75, 112, 256, 512, RELU),
    ("conv4_2", 32, 75, 112, 512, 512, RELU),
    ("conv4_3", 32, 75, 112, 512, 512, RELU | POOL | STACK_OUT),
    ("conv5_1", 32, 37, 56, 512, 512, RELU | STACK_IN | STACK_OUT),
    ("conv5_2", 32, 37, 56, 512, 512, RELU | STACK_IN | STACK_OUT),
    ("conv5_3", 32, 37, 56, 512, 512, RELU | STACK_IN | STACK_OUT),
    ("rpn_conv", 32, 37, 56, 512, 512, RELU | STACK_IN | OUT_BF16X2),   # OUT_BF16X2: f16f8 only
]
UNITS = {"f16f8": 2, "bf16x2": 3}
PEAK = 989e12
SMI = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"]
COLS = {"plain": {}, "-B": {"CTPN_TC_DEBUG": "1"}, "-A": {"CTPN_TC_DEBUG": "2"}, "-MMA": {"CTPN_TC_DEBUG": "4"},
        "-epi": {"CTPN_TC_DEBUG": "16"}, "-epi-st": {"CTPN_TC_DEBUG": "24"}}


def child(mode, reps):
    sys.path.insert(0, os.path.join(ROOT, "text-detection-ctpn_b200"))
    import torch
    from ctpn_b200 import _native as N
    assert N.DEBUG_LIB, "needs the test library (CTPN_B200_LIB=dbg)"
    dev = torch.device("cuda", 0)
    res = {}
    for name, B, H, W, cin, cout, flags in SHAPES:
        if mode != "f16f8":
            flags &= ~OUT_BF16X2
        hin = B * (H + 1) if flags & STACK_IN else B * H
        pool = bool(flags & POOL)
        ho, wo = (H // 2, W // 2) if pool else (H, W)
        hout = B * (ho + 1) if flags & STACK_OUT else B * ho
        g = torch.Generator(device=dev).manual_seed(0)
        x = torch.randint(0, 60, (2 * hin * W * cin * 2,), dtype=torch.uint8, device=dev, generator=g)   # small positive operands
        w = torch.randint(0, 60, (2 * cout * 9 * cin * 2,), dtype=torch.uint8, device=dev, generator=g)
        b = torch.zeros(cout, dtype=torch.float32, device=dev)
        out = torch.empty(2 * hout * wo * cout * 2, dtype=torch.uint8, device=dev)

        def run():
            if mode == "f16f8":
                N.check(N.lib.ctpn_conv3x3_f16f8(N.ptr(x), N.ptr(w), N.ptr(b), N.ptr(out), B, H, W, cin, cout, 9, flags,
                                                 1.0, 1.0, 1.0, 1.0, N.stream_ptr()), "conv")
            else:
                N.check(N.lib.ctpn_conv3x3(N.ptr(x), N.ptr(w), N.ptr(b), N.ptr(out), B, H, W, cin, cout, 9, 2, flags,
                                           N.stream_ptr()), "conv")
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        res[name] = dict(ms=ts[len(ts) // 2], min=ts[0])
        del x, w, out
    card = subprocess.run(SMI + ["-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(mode=mode, card=card, torch_name=torch.cuda.get_device_name(0), shapes=res)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="f16f8,bf16x2")
    ap.add_argument("--cols", default="plain,-MMA,-epi,-epi-st", help="comma-separated columns: " + ",".join(COLS))
    ap.add_argument("--stages-b", default="", help="comma-separated CTPN_TC_STAGES_B values")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--child", default="")
    a = ap.parse_args()
    if a.child:
        child(a.child, a.reps)
        return 0
    cols = [(c, COLS[c]) for c in a.cols.split(",") if c]
    cols += [("sb=%s" % s, {"CTPN_TC_STAGES_B": s}) for s in a.stages_b.split(",") if s]
    print("$ " + " ".join(["python", "tools/conv_pipeline.py"] + sys.argv[1:]))
    for mode in a.modes.split(","):
        table = {}
        for col, env in cols:
            e = {k: v for k, v in os.environ.items() if not k.startswith("CTPN_TC_")}
            e.update(env, CTPN_B200_LIB="dbg")
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", mode, "--reps", str(a.reps)], env=e,
                               capture_output=True, text=True)
            lines = [l for l in p.stdout.splitlines() if l.startswith("{")]
            if p.returncode != 0 or not lines:
                sys.stderr.write(p.stdout[-2000:] + p.stderr[-3000:])
                raise SystemExit("child %s %s failed (exit %d)" % (mode, col, p.returncode))
            table[col] = json.loads(lines[-1])
            print("# %s %-7s card: %s" % (mode, col, table[col]["card"]), flush=True)
        print("\n## %s, batch 32 x 600x900, median ms of %d launches" % (mode, a.reps))
        print("%-8s %7s " % ("layer", "floor") + " ".join("%8s" % c for c, _ in cols))
        for name, B, H, W, cin, cout, flags in SHAPES:
            floor = 2.0 * B * H * W * 9 * cin * cout * UNITS[mode] / PEAK * 1e3
            cells = " ".join("%8.3f" % table[c]["shapes"][name]["ms"] for c, _ in cols)
            print("%-8s %7.3f %s" % (name, floor, cells))
        tot = " ".join("%8.3f" % sum(table[c]["shapes"][s[0]]["ms"] for s in SHAPES) for c, _ in cols)
        fsum = sum(2.0 * B * H * W * 9 * cin * cout * UNITS[mode] / PEAK * 1e3 for _, B, H, W, cin, cout, _ in SHAPES)
        print("%-8s %7.3f %s" % ("sum", fsum, tot))
    return 0


if __name__ == "__main__":
    sys.exit(main())
