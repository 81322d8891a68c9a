"""Head-logit error of several arithmetic modes against the float64 oracle (oracle/net_cpu.py, dtype=torch.float64).

The float32 oracle carries float32 rounding of its own (about 3e-5 on the head logits at 600x900, reported per image as
"f32_oracle"); the float64 oracle takes that out of the comparison.  Per image and mode it prints max|diff|
of rpn_cls_score and rpn_bbox_pred against float64 (and against float32, for the 1e-3 contract), and the card it ran on.

--simt runs the same plane operands through the test library's float32 SIMT convolutions and matmuls (fmaf, round to
nearest) instead of the wgmma kernels; set against a run without it, that separates the operand format's error from the
tensor core's truncating float32 accumulation (DESIGN.md §5).

    python tools/head_error_f64.py --modes bf16x2,bf16x3,f16f8 --seeds 11-16 --out head_f64.json
    python tools/head_error_f64.py --modes bf16x2,bf16x3 --simt --out head_f64_simt.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, "text-detection-ctpn_b200"), ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def parse_seeds(s):
    if "-" in s:
        lo, hi = s.split("-")
        return list(range(int(lo), int(hi) + 1))
    return [int(x) for x in s.split(",")]


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="bf16x2,bf16x3,f16f8")
    ap.add_argument("--seeds", default="11-16")
    ap.add_argument("--H", type=int, default=600)
    ap.add_argument("--W", type=int, default=900)
    ap.add_argument("--simt", action="store_true", help="float32 SIMT convolutions of the test library instead of wgmma")
    ap.add_argument("--out", default=None, help="write the JSON record here as well")
    ap.add_argument("--dry-run", action="store_true", help="parse arguments and exit (no GPU, no oracle)")
    a = ap.parse_args(argv)
    modes, seeds = a.modes.split(","), parse_seeds(a.seeds)
    if a.simt and "f16f8" in modes:
        ap.error("--simt: the SIMT reference kernels read bf16 planes only")
    if a.dry_run:
        print(json.dumps({"modes": modes, "seeds": seeds, "H": a.H, "W": a.W, "simt": a.simt, "out": a.out}))
        return None
    if a.simt:
        os.environ["CTPN_B200_LIB"] = "dbg"        # read when ctpn_b200 is first imported
    import numpy as np
    import torch
    from ctpn_b200 import Engine
    from oracle import net_cpu, synth
    w = synth.make_weights(0)
    engines = {m: Engine(w, mode=m, conv_simt=a.simt) for m in modes}
    rec = {"card": card(), "H": a.H, "W": a.W, "oracle": "float64", "convolutions": "simt" if a.simt else "wgmma",
           "images": []}
    for seed in seeds:
        im = synth.make_image(seed, a.H, a.W)
        blob, scale = net_cpu.image_blob(im)
        assert scale == 1.0
        t0 = time.time()
        r64 = net_cpu.forward(blob, w, dtype=torch.float64)
        r32 = net_cpu.forward(blob, w)
        row = {"seed": seed, "oracle_s": round(time.time() - t0, 1)}
        for m, eng in engines.items():
            cls, box = eng.forward_heads(torch.from_numpy(im[None]).cuda())
            cls, box = cls.cpu().numpy().astype(np.float64), box.cpu().numpy().astype(np.float64)
            row[m] = {"cls_f64": float(np.abs(cls - r64["rpn_cls_score"]).max()),
                      "box_f64": float(np.abs(box - r64["rpn_bbox_pred"]).max()),
                      "cls_f32": float(np.abs(cls - r32["rpn_cls_score"]).max()),
                      "box_f32": float(np.abs(box - r32["rpn_bbox_pred"]).max())}
        row["f32_oracle"] = {"cls_f64": float(np.abs(r32["rpn_cls_score"] - r64["rpn_cls_score"]).max()),
                             "box_f64": float(np.abs(r32["rpn_bbox_pred"] - r64["rpn_bbox_pred"]).max())}
        rec["images"].append(row)
        print("seed %d  " % seed + "  ".join("%s cls %.2e box %.2e" % (m, row[m]["cls_f64"], row[m]["box_f64"])
                                             for m in modes + ["f32_oracle"]), flush=True)
    for m in modes + ["f32_oracle"]:
        rec[m + "_max_cls_f64"] = max(r[m]["cls_f64"] for r in rec["images"])
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)
    return rec


if __name__ == "__main__":
    main()
