"""Line crops out of the source photos (crop_from="source") against crops out of the resize_im canvas and against cutting
source crops on the host.  Legs, alternating in one process, medians (min, max) of the rounds, all through
stream_lines_images with batches of up to --max-batch images:
  canvas  crop_height=Hc: crops cut on the device from the 600-px canvas the lines were found on;
  source  crop_height=Hc, crop_from="source": crops cut on the device from the source at full resolution;
  diy     the lines only, then per image the source brought to the host (a tensor or frame copied back, a YUV frame
          converted with cv2.cvtColor), per line cv2.warpAffine of the source with the crop recipe on lines / f, and the
          padded crops uploaded with torch -- what a user writes without crop_from="source".
source and diy give the same crops bit for bit (asserted).  Workloads: the 64 mixed photos of time_frontend.py as host
arrays and as BGR CUDA tensors, 32 x 3024x4032 BGR tensors and 64 x 3840x2160 NV12 frames.  Synthetic weights score
low, so the connector runs with lowered score thresholds (LOW) to give the photos lines.  Reported per workload and Hc:
images/s, lines per image, H2D and D2H bytes per image from a torch.profiler census of one run per leg, and the crop
kernel's ms per batch from the library's CUDA-event profile.  The card's name and power limit are read in the same run.

    python tools/time_source_crops.py --rounds 5 --out profiles/source_crops_h100.json
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
from time_line_crops import census  # noqa: E402

LOW = (0.05, 0.2, 50, 0.5, 0.5, 0.0, 0.0, 16, 2)
LEGS = ("canvas", "source", "diy")
KERNELS = ("line_crops_u8", "line_crops_strided_u8", "line_crops_yuv420_u8")


def host_source(im):
    """The source of one image as a host BGR array (a tensor or frame copied back)."""
    import cv2
    import torch
    from ctpn_b200 import YUV420
    if isinstance(im, YUV420):
        h, w = im.shape[:2]
        i420 = np.concatenate([im.y.cpu().numpy().ravel(), im.u.cpu().numpy().ravel(), im.v.cpu().numpy().ravel()])
        return cv2.cvtColor(i420.reshape(h * 3 // 2, w), cv2.COLOR_YUV2BGR_I420)
    return im.cpu().numpy() if torch.is_tensor(im) else im


def host_crops(src, lines, f, hc):
    """The source crops of one image's lines, cut with cv2 on the host: (uint8 [m, hc, Wmax, 3], int64 widths [m])."""
    import cv2
    from oracle.crop import crop_matrix, crop_widths
    sl = np.array(lines, np.float64).reshape(-1, 9)
    sl[:, :8] /= np.float64(f)
    widths = crop_widths(sl, hc)
    out = np.zeros((len(sl), hc, int(widths.max()) if len(sl) else 0, 3), np.uint8)
    for j, ln in enumerate(sl):
        out[j, :, :widths[j]] = cv2.warpAffine(src, crop_matrix(ln, hc, widths[j]), (int(widths[j]), hc),
                                               flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP, borderMode=cv2.BORDER_REPLICATE)
    return out, widths


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="f16f8")
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--heights", default="32,48")
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds per workload (at least 3)")
    ap.add_argument("--out", default=None, help="write the JSON record here as well")
    a = ap.parse_args(argv)

    import cv2
    import torch
    from ctpn_b200 import YUV420, Engine, _native as N
    from ctpn_b200.synthetic import make_image, make_weights
    assert a.rounds >= 3, "at least 3 rounds"
    eng = Engine(make_weights(0), mode=a.mode)            # raises without a GPU: there is nothing to time on a CPU
    rec = {"tool": "time_source_crops", "max_batch": a.max_batch, "mode": a.mode, "rounds": a.rounds, "low_cfg": LOW,
           "card": card(), "device": torch.cuda.get_device_name(0)}
    photos = [make_image(i, h, w) for i, (h, w) in enumerate(workload(64))]
    eng.rois_images(photos[:8], max_batch=8)              # F16F8 calibrates on real-sized images
    cams = [make_image(3000 + i, 3024, 4032) for i in range(32)]
    frames = []
    for i in range(64):
        bgr = make_image(4000 + i, 2160, 3840)
        frames.append(YUV420.from_buffer(torch.from_numpy(cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)).cuda(), "NV12"))
    workloads = {"photos64_host_stream": photos, "photos64_bgr_tensors": [torch.from_numpy(p).cuda() for p in photos],
                 "camera32_3024x4032_bgr_tensors": [torch.from_numpy(p).cuda() for p in cams],
                 "video64_3840x2160_nv12": frames}
    del cams
    kw = dict(mode="H", max_batch=a.max_batch, cfg=LOW)

    def leg(ims, hc, name):
        if name == "diy":
            out = []
            for (lines, f), im in zip(eng.stream_lines_images(iter(ims), **kw), ims):
                crops, widths = host_crops(host_source(im), lines, f, hc)
                out.append((lines, torch.from_numpy(crops).to(eng.device), widths))
            return out
        crop_from = "resized" if name == "canvas" else "source"
        return [(lines, crops, widths) for lines, f, crops, widths in
                eng.stream_lines_images(iter(ims), crop_height=hc, crop_from=crop_from, **kw)]

    def crop_kernel(ims, hc, name):
        torch.cuda.synchronize()
        N.check(N.lib.ctpn_prof_enable(1), "ctpn_prof_enable")       # a run of its own: events bracket every launch
        leg(ims, hc, name)
        torch.cuda.synchronize()
        got = {e["kernel"]: e for e in N.prof_report() if e["kernel"] in KERNELS}
        N.check(N.lib.ctpn_prof_enable(0), "ctpn_prof_enable")
        return {k: {"launches": e["launches"], "ms_per_batch": round(e["ms"] / max(1, e["launches"]), 5)} for k, e in got.items()}

    rec["workloads"] = {}
    for wname, ims in workloads.items():
        for hc in (int(h) for h in a.heights.split(",")):
            legs = {k: (lambda k=k: leg(ims, hc, k)) for k in LEGS}
            ref = {}
            for k, f in legs.items():          # warm-up; source and diy give the same crops
                f()
                ref[k] = f()
            for (l1, c1, w1), (l2, c2, w2), (l3, _, _) in zip(ref["source"], ref["diy"], ref["canvas"]):
                assert np.array_equal(l1, l2) and np.array_equal(l1, l3) and np.array_equal(w1, w2) and torch.equal(c1, c2)
            m = len(ims)
            wall = {k: [] for k in legs}
            for r in range(a.rounds):
                for k in (LEGS if r % 2 == 0 else LEGS[::-1]):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    legs[k]()
                    torch.cuda.synchronize()
                    wall[k].append(time.perf_counter() - t0)
            res = {"images": m, "crop_height": hc, "lines_per_image": round(sum(len(x[0]) for x in ref["source"]) / m, 2)}
            for k in legs:
                ips = [m / t for t in wall[k]]
                h2d, d2h = census(legs[k], lambda: eng.detect_lines_images(photos[:2], **kw))
                res[k] = {"images_per_s_median": round(float(np.median(ips)), 2), "min": round(float(min(ips)), 2),
                          "max": round(float(max(ips)), 2), "h2d_bytes_per_image_census": round(h2d / m, 1),
                          "d2h_bytes_per_image_census": round(d2h / m, 1)}
                if k != "diy":
                    res[k]["crop_kernel"] = crop_kernel(ims, hc, k)
            res["source_over_canvas_median"] = round(res["source"]["images_per_s_median"] / res["canvas"]["images_per_s_median"], 3)
            res["source_over_diy_median"] = round(res["source"]["images_per_s_median"] / res["diy"]["images_per_s_median"], 3)
            rec["workloads"]["%s_hc%d" % (wname, hc)] = res
            print(json.dumps({wname: res}), flush=True)
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
