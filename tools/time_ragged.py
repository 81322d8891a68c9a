"""Images/s of mixed-size input: today's shape bucketing (Engine.detect_list) against ragged batches (Engine.detect_ragged)
and against uniform batches of the same canvas shapes, plus a ragged-vs-plain pair at full extents that isolates the cost of
the extent masking.  The workload is 64 seeded photo sizes in both orientations taken through the demo's resize_im (short
side 600, long side <= 1200) and _get_image_blob's scale rule (long side <= MAX_SIZE = 1000), as synthetic uint8 images of
those blob sizes.  All legs alternate in one process (at least 5 rounds, medians and spread); the card's name and power limit
are read in the same run.

    python tools/time_ragged.py --modes f16f8,bf16x2 --rounds 5 --out profiles/ragged_h100.json
    python tools/time_ragged.py --dry-run          # the workload and its batches, no GPU
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

import numpy as np  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def blob_sizes(n, seed=0):
    """n photo sizes (both orientations) -> the blob (h, w) and im_scale the demo feeds the network."""
    from ctpn_b200 import _native as N
    import ctypes as C
    rs = np.random.RandomState(seed)
    out = []
    for i in range(n):
        long_side = int(rs.randint(640, 4033))
        short = int(round(long_side / rs.uniform(1.0, 2.4)))
        h, w = (short, long_side) if i % 2 == 0 else (long_side, short)
        f = 600.0 / min(h, w)                                  # resize_im(im, 600, 1200), ctpn/demo.py
        if f * max(h, w) > 1200:
            f = 1200.0 / max(h, w)
        dh, dw = C.c_int(), C.c_int()
        N.check(N.lib.ctpn_resize_out_size(h, w, f, f, C.byref(dh), C.byref(dw)), "ctpn_resize_out_size")
        h, w = dh.value, dw.value
        s = 600.0 / min(h, w)                                  # _get_image_blob (lib/fast_rcnn/test.py)
        if np.round(s * max(h, w)) > 1000:
            s = 1000.0 / max(h, w)
        N.check(N.lib.ctpn_resize_out_size(h, w, s, s, C.byref(dh), C.byref(dw)), "ctpn_resize_out_size")
        out.append(((dh.value, dw.value), s))
    return out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="f16f8,bf16x2")
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds (at least 5)")
    ap.add_argument("--mask-batch", type=int, default=32, help="batch of the full-extent ragged-vs-plain pair (600 x 1000)")
    ap.add_argument("--out", default=None, help="write the JSON record here as well")
    ap.add_argument("--dry-run", action="store_true", help="print the workload and its batches only (no GPU)")
    a = ap.parse_args(argv)
    from ctpn_b200.engine import ragged_plan
    work = blob_sizes(a.images)
    shapes = [s for s, _ in work]
    plan = ragged_plan(shapes, ["|u1"] * len(shapes), a.max_batch)
    real = sum(h * w for h, w in shapes)
    canvas = sum(len(idx) * H * W for idx, (H, W) in plan)
    rec = {"tool": "time_ragged", "images": len(shapes), "max_batch": a.max_batch, "distinct_shapes": len(set(shapes)),
           "batches": [[len(idx), H, W] for idx, (H, W) in plan], "padded_fraction": round(1.0 - real / canvas, 4),
           "landscape": sum(1 for h, w in shapes if h <= w)}
    if a.dry_run:
        rec["dry_run"] = True
        print(json.dumps(rec))
        return rec

    import torch
    from ctpn_b200 import Engine
    from ctpn_b200.synthetic import make_image, make_weights
    assert a.rounds >= 5, "at least 5 rounds"
    rec["card"] = card()
    rec["device"] = torch.cuda.get_device_name(0)
    images = [make_image(i, h, w) for i, (h, w) in enumerate(shapes)]
    scales = [s for _, s in work]
    weights = make_weights(0)
    rec["modes"] = {}
    for mode in a.modes.split(","):
        eng = Engine(weights, mode=mode)
        eng.detect_ragged(images[:4], max_batch=4)                 # calibrates F16F8 on real-sized images
        canvases = [(np.stack([np.zeros((H, W, 3), np.uint8)] * len(idx)), len(idx)) for idx, (H, W) in plan]
        mb = np.stack([make_image(7, 600, 1000)] * a.mask_batch)
        dev = torch.from_numpy(mb).cuda()
        info = torch.tensor([[600, 1000, 1.0]] * a.mask_batch, dtype=torch.float32, device="cuda")
        full = [(600, 1000)] * a.mask_batch

        def leg_list():
            eng.detect_list(images, max_batch=a.max_batch)
            return len(images)

        def leg_ragged():
            eng.detect_ragged(images, im_scales=scales, max_batch=a.max_batch)
            return len(images)

        def leg_uniform():
            for c, _ in canvases:
                eng.detect_batch(c)
            return len(images)

        def leg_plain():
            eng.detect_packed(dev, info)
            return a.mask_batch

        def leg_full_extent():
            eng.detect_packed(dev, info, sizes=full)
            return a.mask_batch

        legs = {"detect_list": leg_list, "detect_ragged": leg_ragged, "uniform_same_canvases": leg_uniform,
                "plain_600x1000": leg_plain, "ragged_full_extent_600x1000": leg_full_extent}
        for f in legs.values():      # warm-up: weights, workspaces, attribute and tensor-map caches, graph buckets
            f()
            f()
        torch.cuda.synchronize()
        times = {k: [] for k in legs}
        for r in range(a.rounds):
            order = list(legs) if r % 2 == 0 else list(legs)[::-1]
            for k in order:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                n = legs[k]()
                torch.cuda.synchronize()
                times[k].append(n / (time.perf_counter() - t0))
        rec["modes"][mode] = {k: {"images_per_s_median": round(float(np.median(v)), 2), "min": round(float(min(v)), 2),
                                  "max": round(float(max(v)), 2)} for k, v in times.items()}
        rec["modes"][mode]["detect_list"]["padded_fraction"] = 0.0
        rec["modes"][mode]["detect_ragged"]["padded_fraction"] = rec["padded_fraction"]
        rec["modes"][mode]["uniform_same_canvases"]["padded_fraction"] = rec["padded_fraction"]
        del eng
        torch.cuda.empty_cache()
    rec["card_after"] = card()
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    return rec


if __name__ == "__main__":
    main()
