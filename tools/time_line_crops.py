"""Text-line crops for a recognizer: cut on the device against cut on the host.  Legs, alternating in one process, medians
of the rounds:
  host    detect_lines_images(..., return_resized=True), then per line cv2.warpAffine of the resize_im output with the
          crop recipe (include/ctpn_b200.h) at height 32, each image's crops padded into one [m, 32, Wmax, 3] array and
          uploaded with torch (what a user writes without crop_height);
  device  detect_lines_images(..., crop_height=32): the crops are cut on the device from the canvas the lines came from.
Both legs give the same lines and the same crops bit for bit (asserted).  Workloads: the 64 photos of time_frontend.py
and 32 x 600x900 as host arrays, and the 64 photos as BGR CUDA tensors.  Synthetic weights score low, so the connector
runs with lowered score thresholds (LOW) to give the photos lines.  Reported per workload: images/s (median, min, max),
lines per image, H2D and D2H bytes per image from a torch.profiler census of one run per leg, and the crop kernel's ms
per batch from the library's CUDA-event profile.  The card's name and power limit are read in the same run.

    python tools/time_line_crops.py --rounds 5 --out profiles/line_crops_h100.json
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

HC = 32
LOW = (0.05, 0.2, 50, 0.5, 0.5, 0.0, 0.0, 16, 2)
LEGS = ("host", "device")


def host_crops(resized, lines):
    """The crops of one image's lines, cut with cv2 on the host: (uint8 [m, HC, Wmax, 3], int64 widths [m])."""
    import cv2
    from oracle.crop import crop_matrix, crop_widths
    widths = crop_widths(lines, HC)
    out = np.zeros((len(lines), HC, int(widths.max()) if len(lines) else 0, 3), np.uint8)
    for j, ln in enumerate(lines):
        out[j, :, :widths[j]] = cv2.warpAffine(resized, crop_matrix(ln, HC, widths[j]), (int(widths[j]), HC),
                                               flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP, borderMode=cv2.BORDER_REPLICATE)
    return out, widths


def census(fn, warm):
    """(H2D bytes, D2H bytes) of one run of fn, from a torch.profiler trace (warm() runs first inside the profile: the
    profiler can lose the first device records after it starts)."""
    import tempfile
    import torch
    from torch.profiler import ProfilerActivity, profile, record_function
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        warm()
        torch.cuda.synchronize()
        with record_function("census_run"):
            fn()
            torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    span = next(e for e in events if e.get("name") == "census_run" and e.get("cat") == "user_annotation")
    t0, t1 = span["ts"], span["ts"] + span["dur"]
    copies = [e for e in events if e.get("cat") == "gpu_memcpy" and t0 <= e.get("ts", -1) <= t1]
    return tuple(sum(int(e.get("args", {}).get("bytes", 0)) for e in copies if kind in e["name"]) for kind in ("HtoD", "DtoH"))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="f16f8")
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds per workload (at least 3)")
    ap.add_argument("--out", default=None, help="write the JSON record here as well")
    a = ap.parse_args(argv)

    import torch
    from ctpn_b200 import Engine, _native as N
    from ctpn_b200.synthetic import make_image, make_weights
    assert a.rounds >= 3, "at least 3 rounds"
    eng = Engine(make_weights(0), mode=a.mode)            # raises without a GPU: there is nothing to time on a CPU
    rec = {"tool": "time_line_crops", "crop_height": HC, "max_batch": a.max_batch, "mode": a.mode, "rounds": a.rounds,
           "low_cfg": LOW, "card": card(), "device": torch.cuda.get_device_name(0)}
    photos = [make_image(i, h, w) for i, (h, w) in enumerate(workload(64))]
    eng.rois_images(photos[:8], max_batch=8)              # F16F8 calibrates on real-sized images
    workloads = {"photos64": photos, "synthetic32_600x900": [make_image(1000 + i, 600, 900) for i in range(32)],
                 "photos64_bgr_tensors": [torch.from_numpy(p).cuda() for p in photos]}
    kw = dict(mode="H", max_batch=a.max_batch, cfg=LOW)

    def leg_host(ims):
        out = []
        for lines, f, resized in eng.detect_lines_images(ims, return_resized=True, **kw):
            crops, widths = host_crops(resized, lines)
            out.append((lines, torch.from_numpy(crops).to(eng.device), widths))
        return out

    def leg_device(ims):
        return [(lines, crops, widths) for lines, f, crops, widths in eng.detect_lines_images(ims, crop_height=HC, **kw)]

    def crop_kernel(ims):
        torch.cuda.synchronize()
        N.check(N.lib.ctpn_prof_enable(1), "ctpn_prof_enable")       # a run of its own: events bracket every launch
        leg_device(ims)
        torch.cuda.synchronize()
        got = {e["kernel"]: e for e in N.prof_report() if e["kernel"] == "line_crops_u8"}
        N.check(N.lib.ctpn_prof_enable(0), "ctpn_prof_enable")
        e = got.get("line_crops_u8", {"launches": 0, "ms": 0.0})
        return {"launches": e["launches"], "ms_per_batch": round(e["ms"] / max(1, e["launches"]), 5)}

    rec["workloads"] = {}
    for name, ims in workloads.items():
        legs = {"host": lambda: leg_host(ims), "device": lambda: leg_device(ims)}
        assert tuple(legs) == LEGS
        ref = None
        for k, f in legs.items():          # warm-up; both legs give the same lines and crops
            f()
            out = f()
            ref = out if ref is None else ref
            assert len(out) == len(ref), k
            for (l1, c1, w1), (l2, c2, w2) in zip(out, ref):
                assert np.array_equal(l1, l2) and np.array_equal(w1, w2) and torch.equal(c1, c2), k
        m = len(ims)
        wall = {k: [] for k in legs}
        for r in range(a.rounds):
            for k in (LEGS if r % 2 == 0 else LEGS[::-1]):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                legs[k]()
                torch.cuda.synchronize()
                wall[k].append(time.perf_counter() - t0)
        res = {"images": m, "lines_per_image": round(sum(len(x[0]) for x in ref) / m, 2)}
        for k in legs:
            ips = [m / t for t in wall[k]]
            h2d, d2h = census(legs[k], lambda: eng.detect_lines_images(ims[:2], **kw))
            res[k] = {"images_per_s_median": round(float(np.median(ips)), 2), "min": round(float(min(ips)), 2),
                      "max": round(float(max(ips)), 2), "h2d_bytes_per_image_census": round(h2d / m, 1),
                      "d2h_bytes_per_image_census": round(d2h / m, 1)}
        res["speedup_median"] = round(res["device"]["images_per_s_median"] / res["host"]["images_per_s_median"], 3)
        res["crop_kernel"] = crop_kernel(ims)
        rec["workloads"][name] = res
        print(json.dumps({name: res}), flush=True)
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
