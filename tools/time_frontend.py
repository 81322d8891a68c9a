"""Host front-end against device front-end for a folder of photos.  (a) what ctpn/demo.py --batch does: cv2 resize_im and
_get_image_blob per image on the host, then Engine.rois_ragged on the blobs; (b) Engine.rois_images on the raw images
(resize_im and the blob on the device, one H2D of the packed sources per batch).  The workload is 64 seeded synthetic
uint8 photos of the sizes a user's folder holds (480x640, 768x1024, 1080x1920, 3024x4032, 1000x3000), both orientations;
the 3:1 and 16:9 ones are wider than 5:3, so their blobs take _get_image_blob's float32 rescale.  Both legs alternate in
one process, on the whole workload and on each source size alone; reported: images/s, host CPU seconds per image
(time.process_time, all threads), H2D bytes per image computed from shapes, and the two ragged kernels' times from
ctpn_prof.  The card's name and power limit are read in the same run.

    python tools/time_frontend.py --rounds 5 --out profiles/frontend_h100.json
    python tools/time_frontend.py --dry-run          # the workload, its batches and H2D bytes, no GPU
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

SIZES = [(480, 640), (768, 1024), (1080, 1920), (3024, 4032), (1000, 3000)]


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def workload(n, seed=0):
    """n photo shapes: the five sizes in turn, orientation seeded (about half portrait)."""
    rs = np.random.RandomState(seed)
    out = []
    for i in range(n):
        h, w = SIZES[i % len(SIZES)]
        out.append((w, h) if rs.rand() < 0.5 else (h, w))
    return out


def h2d_bytes(shapes, max_batch):
    """Bytes each leg uploads: (a) rois_ragged copies every batch's padded blob canvas (uint8 or float32); (b) rois_images
    copies the packed uint8 sources."""
    from ctpn_b200.engine import frontend_plan, ragged_plan
    plan = frontend_plan(shapes)
    host = 0
    for idxs, (H, W) in ragged_plan([p.blob for p in plan], [p.dtype for p in plan], max_batch):
        host += len(idxs) * H * W * 3 * (1 if plan[idxs[0]].dtype == "|u1" else 4)
    return host, sum(h * w * 3 for h, w in shapes), plan


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="f16f8")
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds per comparison (at least 3)")
    ap.add_argument("--out", default=None, help="write the JSON record here as well")
    ap.add_argument("--dry-run", action="store_true", help="print the workload, its batches and H2D bytes only (no GPU)")
    a = ap.parse_args(argv)
    from ctpn_b200.engine import ragged_plan
    shapes = workload(a.images)
    host_b, dev_b, plan = h2d_bytes(shapes, a.max_batch)
    n = len(shapes)
    rec = {"tool": "time_frontend", "images": n, "max_batch": a.max_batch, "mode": a.mode,
           "sizes": {"%dx%d" % s: sum(1 for h, w in shapes if (h, w) in (s, s[::-1])) for s in SIZES},
           "float_blobs": sum(1 for p in plan if p.dtype == "<f4"),
           "batches_device": [[len(i), H, W] for i, (H, W) in ragged_plan([p.blob for p in plan], [p.dtype for p in plan], a.max_batch)],
           "h2d_bytes_per_image": {"host_frontend": round(host_b / n), "device_frontend": round(dev_b / n)}}
    if a.dry_run:
        rec["dry_run"] = True
        print(json.dumps(rec))
        return rec

    import torch
    from ctpn import demo
    from ctpn_b200 import Engine, _native as N
    from ctpn_b200.synthetic import make_image, make_weights
    from lib.fast_rcnn.test import _get_image_blob
    assert a.rounds >= 3, "at least 3 rounds"
    rec["card"] = card()
    rec["device"] = torch.cuda.get_device_name(0)
    images = [make_image(i, h, w) for i, (h, w) in enumerate(shapes)]
    eng = Engine(make_weights(0), mode=a.mode)
    eng.rois_images(images[:8], max_batch=8)                  # F16F8 calibrates on real-sized images

    def leg_host(ims):
        blobs, scales = [], []
        for im in ims:
            img, _ = demo.resize_im(im, scale=600, max_scale=1200)
            blob, im_scale = _get_image_blob(img)
            blobs.append(blob[0])
            scales.append(float(im_scale[0]))
        eng.rois_ragged(blobs, im_scales=scales, max_batch=a.max_batch)

    def leg_device(ims):
        eng.rois_images(ims, max_batch=a.max_batch)

    legs = {"host_frontend": leg_host, "device_frontend": leg_device}

    def compare(ims):
        for f in legs.values():      # warm-up: workspaces, pinned buffers, graph buckets of this subset
            f(ims)
            f(ims)
        wall = {k: [] for k in legs}
        cpu = {k: [] for k in legs}
        for r in range(a.rounds):
            for k in (list(legs) if r % 2 == 0 else list(legs)[::-1]):
                torch.cuda.synchronize()
                t0, c0 = time.perf_counter(), time.process_time()
                legs[k](ims)
                torch.cuda.synchronize()
                wall[k].append(time.perf_counter() - t0)
                cpu[k].append(time.process_time() - c0)
        m = len(ims)
        hb, db, _ = h2d_bytes([im.shape[:2] for im in ims], a.max_batch)
        out = {}
        for k in legs:
            ips = [m / t for t in wall[k]]
            out[k] = {"images_per_s_median": round(float(np.median(ips)), 2), "min": round(float(min(ips)), 2),
                      "max": round(float(max(ips)), 2),
                      "host_cpu_s_per_image_median": round(float(np.median(cpu[k])) / m, 5),
                      "h2d_bytes_per_image": round((hb if k == "host_frontend" else db) / m)}
        return out

    rec["all"] = compare(images)
    rec["per_source_size"] = {}
    for s in SIZES:
        sub = [im for im in images if im.shape[:2] in (s, s[::-1])]
        rec["per_source_size"]["%dx%d" % s] = dict(images=len(sub), **compare(sub))
    torch.cuda.synchronize()
    N.check(N.lib.ctpn_prof_enable(1), "ctpn_prof_enable")        # a run of its own: events bracket every launch
    leg_device(images)
    torch.cuda.synchronize()
    prof = [e for e in N.prof_report() if e["kernel"] in ("resize_linear_u8_ragged", "image_blob_f32_ragged")]
    N.check(N.lib.ctpn_prof_enable(0), "ctpn_prof_enable")
    rec["kernels"] = {e["kernel"]: {"launches": e["launches"], "ms": round(e["ms"], 4), "output_elems": e["work"],
                                    "ms_per_image": round(e["ms"] / n, 5)} for e in prof}
    rec["card_after"] = card()
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    return rec


if __name__ == "__main__":
    main()
