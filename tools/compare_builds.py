#!/usr/bin/env python
"""Byte-for-byte comparison of two builds of the repository: a change that only reschedules kernels must not change a bit.

    python tools/compare_builds.py OLD_ROOT NEW_ROOT [--out DIR]

Each ROOT is a built checkout (libraries in place).  For each, one child process per case writes its outputs under
DIR/<old|new>/<case>/, then every .npy file is compared byte for byte:
    bench.py --dump-outputs: --config 2, 4 and 5 (f16f8), and --config 2 with --mode bf16x2 and --mode bf16 (rois, counts)
    Engine.forward_heads on three seeded 600x900 images in every arithmetic mode (bf16, bf16x2, bf16x3, bf16x3p, f16f8),
    as one batch and, for the ragged path, with per-image sizes (head logits and box deltas)
Exit status 0 when every file is identical.
"""
import argparse
import os
import subprocess
import sys

BENCH_CASES = [("cfg2", ["--config", "2"]), ("cfg4", ["--config", "4"]), ("cfg5", ["--config", "5"]),
               ("cfg2_bf16x2", ["--config", "2", "--mode", "bf16x2"]), ("cfg2_bf16", ["--config", "2", "--mode", "bf16"])]
MODES = ["bf16", "bf16x2", "bf16x3", "bf16x3p", "f16f8"]


def heads_child(root, out):
    sys.path.insert(0, os.path.join(root, "text-detection-ctpn_b200"))
    sys.path.insert(0, root)
    import numpy as np
    import torch
    from ctpn_b200 import Engine
    from oracle import synth
    ims = np.stack([synth.make_image(s, 600, 900) for s in (1, 2, 3)])
    x = torch.from_numpy(ims).cuda()
    sizes = np.array([[600, 900], [480, 700], [352, 544]], np.int32)
    w = synth.make_weights(0)
    os.makedirs(out, exist_ok=True)
    for mode in MODES:
        eng = Engine(w, mode=mode, device=0)
        for tag, kw in (("batch", {}), ("ragged", {"sizes": sizes})):
            cls, box = eng.forward_heads(x, **kw)
            torch.cuda.synchronize()
            np.save(os.path.join(out, "%s_%s_cls.npy" % (mode, tag)), cls.cpu().numpy())
            np.save(os.path.join(out, "%s_%s_box.npy" % (mode, tag)), box.cpu().numpy())
        del eng
        torch.cuda.empty_cache()


def run_build(root, out):
    for name, args in BENCH_CASES:
        d = os.path.join(out, name)
        cmd = [sys.executable, os.path.join(root, "bench.py"), "--gpus", "1", "--steps", "2", "--warmup", "1", "--cpu-sample", "0",
               "--alt-modes", "0", "--dump-outputs", d] + args
        r = subprocess.run(cmd, cwd=root, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout[-2000:] + r.stderr[-3000:])
            raise SystemExit("%s: bench %s failed" % (root, name))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--heads-child", root, os.path.join(out, "heads")],
                       capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-2000:] + r.stderr[-3000:])
        raise SystemExit("%s: forward_heads failed" % root)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("roots", nargs="*")
    ap.add_argument("--out", default="compare_out")
    ap.add_argument("--heads-child", nargs=2, metavar=("ROOT", "OUT"))
    a = ap.parse_args()
    if a.heads_child:
        heads_child(*a.heads_child)
        return 0
    import numpy as np
    old, new = (os.path.abspath(r) for r in a.roots)
    out = os.path.abspath(a.out)
    run_build(old, os.path.join(out, "old"))
    run_build(new, os.path.join(out, "new"))
    bad = n = 0
    for dirpath, _, files in sorted(os.walk(os.path.join(out, "old"))):
        for f in sorted(files):
            if not f.endswith(".npy"):
                continue
            po = os.path.join(dirpath, f)
            rel = os.path.relpath(po, os.path.join(out, "old"))
            x, y = np.load(po), np.load(os.path.join(out, "new", rel))
            same = x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()
            n += 1
            bad += not same
            print("%-9s %-40s %s" % ("identical" if same else "DIFFERENT", rel, x.shape))
    print("%d of %d files identical" % (n - bad, n))
    return 1 if bad or n == 0 else 0


if __name__ == "__main__":
    sys.exit(main())
