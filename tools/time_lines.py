"""Text lines from raw photos: host connector against device connector.  (a) Engine.rois_images, then the library's host
connector (ctpn_text_lines_host, which releases the GIL) for every image on an 8-thread pool, as detect_lines_batches
runs it; (b) Engine.detect_lines_images (the connector kernel on each batch's rois, one D2H of the packed lines); (c) for
scale, the demo's default loop: rois_images, then TextDetector.detect per image in Python (numpy line fit).  Workloads:
the 64 seeded photos of tools/time_frontend.py (five source sizes, both orientations, float32 blob rescales among them)
and 32 synthetic 600x900 images.  The legs alternate in one process; per workload and connector setting: images/s
(median of the rounds, min, max), host CPU seconds per image (time.process_time, all threads), D2H bytes per image
computed from shapes, lines per image, and the connector kernel's time per batch from ctpn_prof.  Synthetic weights
score low, so each workload also runs with the connector thresholds lowered (LOW) to give it chains to build.  The
card's name and power limit are read in the same run.

    python tools/time_lines.py --rounds 5 --out profiles/lines_h100.json
    python tools/time_lines.py --dry-run          # workloads, batches and D2H bytes, no GPU
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, "text-detection-ctpn_b200"), ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402

from time_frontend import card, workload  # noqa: E402

LOW = (0.05, 0.2, 50, 0.5, 0.5, 0.0, 0.0, 0, 0)


def d2h_bytes(rows):
    """Per image: (a) the packed rois + count (float32 [rows][5] + int32); (b) the packed lines + count + status
    (float64 [rows][9] + 2 x int32)."""
    return {"host_connector": rows * 5 * 4 + 4, "device_connector": rows * 9 * 8 + 8}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="f16f8")
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds per comparison (at least 3)")
    ap.add_argument("--out", default=None, help="write the JSON record here as well")
    ap.add_argument("--dry-run", action="store_true", help="print the workloads, their batches and D2H bytes only (no GPU)")
    a = ap.parse_args(argv)
    from ctpn_b200.engine import DEFAULT_CFG, frontend_plan, ragged_plan
    rows = int(DEFAULT_CFG["RPN_POST_NMS_TOP_N"])
    shapes = {"photos64": workload(64), "synthetic32_600x900": [(600, 900)] * 32}
    rec = {"tool": "time_lines", "mode": a.mode, "max_batch": a.max_batch, "workers": a.workers, "rows": rows,
           "d2h_bytes_per_image": d2h_bytes(rows), "workloads": {}}
    for name, sh in shapes.items():
        plan = frontend_plan(sh)
        rec["workloads"][name] = {"images": len(sh), "batches": [[len(i), H, W] for i, (H, W) in
                                                                 ragged_plan([p.blob for p in plan], [p.dtype for p in plan], a.max_batch)]}
    if a.dry_run:
        rec["dry_run"] = True
        print(json.dumps(rec))
        return rec

    import torch
    from concurrent.futures import ThreadPoolExecutor
    from ctpn_b200 import Engine, _native as N
    from ctpn_b200.synthetic import make_image, make_weights
    from ctpn_b200.textlines import text_lines
    from lib.fast_rcnn.config import cfg as rcfg
    from lib.text_connector import text_connect_cfg
    from lib.text_connector.detectors import TextDetector
    assert a.rounds >= 3, "at least 3 rounds"
    rec["card"] = card()
    rec["device"] = torch.cuda.get_device_name(0)
    eng = Engine(make_weights(0), mode=a.mode)
    images = {"photos64": [make_image(i, h, w) for i, (h, w) in enumerate(shapes["photos64"])],
              "synthetic32_600x900": [make_image(1000 + i, 600, 900) for i in range(32)]}
    eng.rois_images(images["photos64"][:8], max_batch=8)          # F16F8 calibrates on real-sized images
    pool = ThreadPoolExecutor(max_workers=a.workers)

    def leg_host(ims, c9):
        res = eng.rois_images(ims, max_batch=a.max_batch)
        plan = frontend_plan(ims)
        futs = [pool.submit(text_lines, r[:, 1:5] / np.float64(s), r[:, 0], p.resized, "H", c9) for (r, s, _), p in zip(res, plan)]
        return [f.result() for f in futs]

    def leg_device(ims, c9):
        return [x[0] for x in eng.detect_lines_images(ims, mode="H", max_batch=a.max_batch, cfg=c9)]

    def leg_python(ims, c9):
        saved = {k: getattr(text_connect_cfg.Config, k) for k in ("TEXT_PROPOSALS_MIN_SCORE", "TEXT_PROPOSALS_NMS_THRESH",
                                                                  "MAX_HORIZONTAL_GAP", "MIN_V_OVERLAPS", "MIN_SIZE_SIM",
                                                                  "MIN_RATIO", "LINE_MIN_SCORE", "TEXT_PROPOSALS_WIDTH",
                                                                  "MIN_NUM_PROPOSALS")}
        try:
            if c9 is not None:
                for k, v in zip(saved, c9):
                    setattr(text_connect_cfg.Config, k, v)
            res = eng.rois_images(ims, max_batch=a.max_batch)
            plan = frontend_plan(ims)
            rcfg.TEST.DETECT_MODE = "H"
            return [TextDetector().detect(r[:, 1:5] / np.float64(s), r[:, 0][:, None], p.resized) for (r, s, _), p in zip(res, plan)]
        finally:
            for k, v in saved.items():
                setattr(text_connect_cfg.Config, k, v)

    legs = {"host_connector_pool": leg_host, "device_connector": leg_device, "python_connector_demo_loop": leg_python}

    def compare(ims, c9):
        outs = {}
        for k, f in legs.items():      # warm-up: workspaces, pinned buffers; and the outputs agree
            f(ims, c9)
            outs[k] = f(ims, c9)
        same = all(np.array_equal(x, y) for x, y in zip(outs["host_connector_pool"], outs["device_connector"]))
        wall = {k: [] for k in legs}
        cpu = {k: [] for k in legs}
        for r in range(a.rounds):
            for k in (list(legs) if r % 2 == 0 else list(legs)[::-1]):
                torch.cuda.synchronize()
                t0, c0 = time.perf_counter(), time.process_time()
                legs[k](ims, c9)
                torch.cuda.synchronize()
                wall[k].append(time.perf_counter() - t0)
                cpu[k].append(time.process_time() - c0)
        m = len(ims)
        out = {"lines_per_image": round(sum(len(x) for x in outs["device_connector"]) / m, 2),
               "device_equals_host_connector": bool(same)}
        for k in legs:
            ips = [m / t for t in wall[k]]
            out[k] = {"images_per_s_median": round(float(np.median(ips)), 2), "min": round(float(min(ips)), 2),
                      "max": round(float(max(ips)), 2),
                      "host_cpu_s_per_image_median": round(float(np.median(cpu[k])) / m, 5)}
        torch.cuda.synchronize()
        N.check(N.lib.ctpn_prof_enable(1), "ctpn_prof_enable")    # a run of its own: events bracket every launch
        leg_device(ims, c9)
        torch.cuda.synchronize()
        prof = [e for e in N.prof_report() if e["kernel"] == "text_lines"]
        N.check(N.lib.ctpn_prof_enable(0), "ctpn_prof_enable")
        if prof:
            e = prof[0]
            out["text_lines_kernel"] = {"launches": e["launches"], "ms_total": round(e["ms"], 4),
                                        "ms_per_batch": round(e["ms"] / e["launches"], 4), "ms_per_image": round(e["ms"] / m, 5)}
        return out

    for name, ims in images.items():
        for label, c9 in (("default_cfg", None), ("low_cfg", LOW)):
            rec["workloads"][name][label] = compare(ims, c9)
    rec["low_cfg"] = LOW
    rec["card_after"] = card()
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    return rec


if __name__ == "__main__":
    main()
