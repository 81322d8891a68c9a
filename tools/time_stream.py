"""Streamed device pipeline against the list calls, for a folder of photos.  Four legs alternate in one process:
(a) host_frontend: what ctpn/demo.py --batch does (cv2 resize_im and _get_image_blob per image on the host, then
Engine.rois_ragged); (b) rois_images: the serial device front-end; (c) stream: Engine.stream_rois_images, sources
row-compacted where that removes a quarter of the rows; (d) stream_dense: the same with compact_rows=False.  The images
are in memory for every leg, so decoding is excluded, as in tools/time_frontend.py, whose workload this is: 64 seeded
synthetic uint8 photos of 480x640, 768x1024, 1080x1920, 3024x4032 and 1000x3000, both orientations, timed as a whole and
per source size.  Reported per leg: images/s (median, min, max of the rounds), host CPU seconds per image
(time.process_time, all threads) and H2D bytes per image computed from shapes; and the time of the row-compacted resize
kernel per batch from the library's CUDA-event profile.  The card's name and power limit are read in the same run.

    python tools/time_stream.py --rounds 5 --out profiles/stream_h100.json
    python tools/time_stream.py --dry-run            # the workload, its batches and H2D bytes, no GPU
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

from time_frontend import SIZES, card, h2d_bytes, workload  # noqa: E402

LEGS = ("host_frontend", "rois_images", "stream", "stream_dense")


def stream_h2d_bytes(shapes, max_batch, window, compact_rows):
    """Bytes stream_rois_images uploads for these (h, w), and how many of its batches carry row maps."""
    from ctpn_b200.engine import frontend_plan, ragged_plan, stream_layout
    total, batches, compacted = 0, 0, 0
    for k in range(0, len(shapes), window):
        part = shapes[k:k + window]
        plan = frontend_plan(part)
        for idxs, _ in ragged_plan([p.blob for p in plan], [p.dtype for p in plan], max_batch):
            lay = stream_layout([plan[i] for i in idxs], [part[i] for i in idxs], compact_rows)
            total += lay.total
            batches += 1
            compacted += lay.maps is not None
    return total, batches, compacted


def leg_bytes(shapes, max_batch, window):
    host_b, dev_b, _ = h2d_bytes(shapes, max_batch)
    return {"host_frontend": host_b, "rois_images": dev_b, "stream": stream_h2d_bytes(shapes, max_batch, window, True)[0],
            "stream_dense": stream_h2d_bytes(shapes, max_batch, window, False)[0]}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="f16f8")
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--window", type=int, default=64, help="images the stream pulls before it plans their batches")
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds per comparison (at least 3)")
    ap.add_argument("--out", default=None, help="write the JSON record here as well")
    ap.add_argument("--dry-run", action="store_true", help="print the workload, its batches and H2D bytes only (no GPU)")
    a = ap.parse_args(argv)
    shapes = workload(a.images)
    n = len(shapes)
    rec = {"tool": "time_stream", "images": n, "max_batch": a.max_batch, "window": a.window, "mode": a.mode,
           "sizes": {"%dx%d" % s: sum(1 for h, w in shapes if (h, w) in (s, s[::-1])) for s in SIZES},
           "stream_batches": dict(zip(("batches", "with_row_maps"), stream_h2d_bytes(shapes, a.max_batch, a.window, True)[1:])),
           "h2d_bytes_per_image": {k: round(v / n) for k, v in leg_bytes(shapes, a.max_batch, a.window).items()}}
    if a.dry_run:
        rec["dry_run"] = True
        rec["h2d_bytes_per_image_per_source_size"] = {
            "%dx%d" % s: {k: round(v / max(1, rec["sizes"]["%dx%d" % s])) for k, v in
                          leg_bytes([x for x in shapes if x in (s, s[::-1])], a.max_batch, a.window).items()} for s in SIZES}
        print(json.dumps(rec))
        return rec

    import torch
    from ctpn import demo
    from ctpn_b200 import Engine, _native as N
    from ctpn_b200.synthetic import make_image, make_weights
    from lib.fast_rcnn.test import _get_image_blob
    assert a.rounds >= 3, "at least 3 rounds"
    eng = Engine(make_weights(0), mode=a.mode)            # raises without a GPU: there is nothing to time on a CPU
    rec["card"] = card()
    rec["device"] = torch.cuda.get_device_name(0)
    images = [make_image(i, h, w) for i, (h, w) in enumerate(shapes)]
    eng.rois_images(images[:8], max_batch=8)                  # F16F8 calibrates on real-sized images

    def leg_host(ims):
        blobs, scales = [], []
        for im in ims:
            img, _ = demo.resize_im(im, scale=600, max_scale=1200)
            blob, im_scale = _get_image_blob(img)
            blobs.append(blob[0])
            scales.append(float(im_scale[0]))
        return eng.rois_ragged(blobs, im_scales=scales, max_batch=a.max_batch)

    legs = {"host_frontend": leg_host,
            "rois_images": lambda ims: [r[0] for r in eng.rois_images(ims, max_batch=a.max_batch)],
            "stream": lambda ims: [r[0] for r in eng.stream_rois_images(iter(ims), max_batch=a.max_batch, window=a.window)],
            "stream_dense": lambda ims: [r[0] for r in eng.stream_rois_images(iter(ims), max_batch=a.max_batch, window=a.window,
                                                                              compact_rows=False)]}
    assert tuple(legs) == LEGS

    def compare(ims):
        ref = None
        for k, f in legs.items():      # warm-up: workspaces, pinned buffers, slot buffers of this subset
            f(ims)
            out = f(ims)
            if k != "host_frontend":   # the device legs must agree bit for bit (the host leg differs where cv2 uses IPP)
                ref = out if ref is None else ref
                assert len(out) == len(ref) and all(np.array_equal(x, y) for x, y in zip(out, ref)), k
        wall = {k: [] for k in legs}
        cpu = {k: [] for k in legs}
        order = list(legs)
        for r in range(a.rounds):
            for k in order[r % len(order):] + order[:r % len(order)]:
                torch.cuda.synchronize()
                t0, c0 = time.perf_counter(), time.process_time()
                legs[k](ims)
                torch.cuda.synchronize()
                wall[k].append(time.perf_counter() - t0)
                cpu[k].append(time.process_time() - c0)
        m = len(ims)
        nbytes = leg_bytes([im.shape[:2] for im in ims], a.max_batch, a.window)
        out = {}
        for k in legs:
            ips = [m / t for t in wall[k]]
            out[k] = {"images_per_s_median": round(float(np.median(ips)), 2), "min": round(float(min(ips)), 2),
                      "max": round(float(max(ips)), 2),
                      "host_cpu_s_per_image_median": round(float(np.median(cpu[k])) / m, 5),
                      "h2d_bytes_per_image": round(nbytes[k] / m)}
        return out

    rec["all"] = compare(images)
    rec["per_source_size"] = {}
    for s in SIZES:
        sub = [im for im in images if im.shape[:2] in (s, s[::-1])]
        rec["per_source_size"]["%dx%d" % s] = dict(images=len(sub), **compare(sub))
    torch.cuda.synchronize()
    N.check(N.lib.ctpn_prof_enable(1), "ctpn_prof_enable")        # a run of its own: events bracket every launch
    legs["stream"](images)
    torch.cuda.synchronize()
    kernels = ("resize_linear_u8_ragged_rows", "resize_linear_u8_ragged", "image_blob_f32_ragged")
    prof = [e for e in N.prof_report() if e["kernel"] in kernels]
    N.check(N.lib.ctpn_prof_enable(0), "ctpn_prof_enable")
    rec["kernels"] = {e["kernel"]: {"launches": e["launches"], "ms": round(e["ms"], 4), "output_elems": e["work"],
                                    "ms_per_batch": round(e["ms"] / max(1, e["launches"]), 5)} for e in prof}
    rec["card_after"] = card()
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    return rec


if __name__ == "__main__":
    main()
