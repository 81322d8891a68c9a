"""Photos already in device memory against the best host path.  The workload of tools/time_stream.py (64 seeded synthetic
photos in five sizes, both orientations), f16f8, batches of up to 32, a window of 64.  Legs, alternating in one process:
  host_stream    host arrays through Engine.stream_rois_images (row-compacted uploads: the best host path so far);
  device_list    CUDA tensors through Engine.rois_images;
  device_stream  CUDA tensors through Engine.stream_rois_images;
and end to end from JPEG bytes (the same photos, blurred so that they compress like photos, encoded by cv2 at quality 90):
  jpeg_host      cv2.imdecode of each file, lazily, into the host stream;
  jpeg_device    torchvision.io.decode_jpeg(device="cuda") (nvJPEG) of each file, lazily, into the device stream.
The device legs take the tensors as a decoder returns them: RGB, planar (chw.permute(1, 2, 0)), channels="RGB".
Reported for the whole workload and per source size: images/s (median, min and max of the rounds), host CPU ms per image
(time.process_time, all threads) and H2D bytes per image -- from shapes where the layout gives them, and from a
torch.profiler census of one run of each leg, made after the timed rounds --, and the resize kernels' ms per batch from
the library's CUDA-event profile (the strided kernel of device_stream beside the dense kernel of host_stream with
compact_rows=False), also after the timed rounds.  The card's name and power limit are read in the same run.

    python tools/time_device_images.py --rounds 5 --out profiles/device_images_h100.json
    python tools/time_device_images.py --dry-run            # the workload and the H2D bytes from shapes, no GPU
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, "text-detection-ctpn_b200"), ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402

from time_frontend import SIZES, card, workload  # noqa: E402
from time_stream import stream_h2d_bytes  # noqa: E402

LEGS = ("host_stream", "device_list", "device_stream", "jpeg_host", "jpeg_device")


def shape_bytes(shapes, max_batch, window):
    """H2D bytes the layouts give for these (h, w): the host stream's uploads, the device stream's sizes / im_info tails."""
    return {"host_stream": stream_h2d_bytes(shapes, max_batch, window, True)[0], "device_stream": 28 * len(shapes)}


def census_h2d(fn):
    """Bytes of every host-to-device copy of one run of fn, from a torch.profiler trace."""
    from torch.profiler import ProfilerActivity, profile
    import torch
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    return sum(int(e.get("args", {}).get("bytes", 0)) for e in events if e.get("cat") == "gpu_memcpy" and "HtoD" in e["name"])


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="f16f8")
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--window", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds per comparison (at least 3)")
    ap.add_argument("--out", default=None, help="write the JSON record here as well")
    ap.add_argument("--dry-run", action="store_true", help="print the workload and the H2D bytes from shapes only (no GPU)")
    a = ap.parse_args(argv)
    shapes = workload(a.images)
    n = len(shapes)
    rec = {"tool": "time_device_images", "images": n, "max_batch": a.max_batch, "window": a.window, "mode": a.mode,
           "sizes": {"%dx%d" % s: sum(1 for h, w in shapes if (h, w) in (s, s[::-1])) for s in SIZES},
           "h2d_bytes_per_image_from_shapes": {k: round(v / n) for k, v in shape_bytes(shapes, a.max_batch, a.window).items()}}
    if a.dry_run:
        rec["dry_run"] = True
        print(json.dumps(rec))
        return rec

    import cv2
    import torch
    from torchvision.io import ImageReadMode, decode_jpeg
    from ctpn_b200 import Engine, _native as N
    from ctpn_b200.synthetic import make_image, make_weights
    assert a.rounds >= 3, "at least 3 rounds"
    eng = Engine(make_weights(0), mode=a.mode)            # raises without a GPU: there is nothing to time on a CPU
    rec["card"] = card()
    rec["device"] = torch.cuda.get_device_name(0)
    images = [make_image(i, h, w) for i, (h, w) in enumerate(shapes)]
    # as a decoder returns them: RGB planes, taken as chw.permute(1, 2, 0)
    tensors = [torch.from_numpy(np.ascontiguousarray(im[:, :, ::-1].transpose(2, 0, 1))).cuda().permute(1, 2, 0) for im in images]
    jpegs = [cv2.imencode(".jpg", cv2.GaussianBlur(im, (0, 0), 2.0), [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes() for im in images]
    eng.rois_images(images[:8], max_batch=8)                  # F16F8 calibrates on real-sized images
    kw = dict(max_batch=a.max_batch, window=a.window)

    def gpu_decoded(ds):
        for d in ds:
            yield decode_jpeg(torch.frombuffer(bytearray(d), dtype=torch.uint8), mode=ImageReadMode.RGB, device="cuda").permute(1, 2, 0)

    legs = {"host_stream": lambda idx: [r[0] for r in eng.stream_rois_images((images[i] for i in idx), **kw)],
            "device_list": lambda idx: [r[0] for r in eng.rois_images([tensors[i] for i in idx], max_batch=a.max_batch,
                                                                      channels="RGB")],
            "device_stream": lambda idx: [r[0] for r in eng.stream_rois_images((tensors[i] for i in idx), channels="RGB", **kw)],
            "jpeg_host": lambda idx: [r[0] for r in eng.stream_rois_images(
                (cv2.imdecode(np.frombuffer(jpegs[i], np.uint8), cv2.IMREAD_COLOR) for i in idx), **kw)],
            "jpeg_device": lambda idx: [r[0] for r in eng.stream_rois_images(gpu_decoded(jpegs[i] for i in idx), channels="RGB",
                                                                             **kw)]}
    assert tuple(legs) == LEGS

    def compare(idx):
        ref = None
        for k, f in legs.items():      # warm-up: workspaces, pinned buffers, slot buffers of this subset
            f(idx)
            out = f(idx)
            if not k.startswith("jpeg"):      # the pixel legs agree bit for bit (the JPEG legs decode different pixels)
                ref = out if ref is None else ref
                assert len(out) == len(ref) and all(np.array_equal(x, y) for x, y in zip(out, ref)), k
        wall = {k: [] for k in legs}
        cpu = {k: [] for k in legs}
        order = list(legs)
        for r in range(a.rounds):
            for k in order[r % len(order):] + order[:r % len(order)]:
                torch.cuda.synchronize()
                t0, c0 = time.perf_counter(), time.process_time()
                legs[k](idx)
                torch.cuda.synchronize()
                wall[k].append(time.perf_counter() - t0)
                cpu[k].append(time.process_time() - c0)
        m = len(idx)
        from_shapes = shape_bytes([shapes[i] for i in idx], a.max_batch, a.window)
        out = {"jpeg_bytes_per_image": round(sum(len(jpegs[i]) for i in idx) / m)}
        for k in legs:
            ips = [m / t for t in wall[k]]
            out[k] = {"images_per_s_median": round(float(np.median(ips)), 2), "min": round(float(min(ips)), 2),
                      "max": round(float(max(ips)), 2), "host_cpu_ms_per_image_median": round(1e3 * float(np.median(cpu[k])) / m, 3)}
            if k in from_shapes:
                out[k]["h2d_bytes_per_image_from_shapes"] = round(from_shapes[k] / m)
        return out

    def kernels(idx):
        """ms per batch of the resize kernels: the dense kernel on whole host images, the strided one on the tensors."""
        got = {}
        for fn in (lambda: eng.stream_rois_images((images[i] for i in idx), compact_rows=False, **kw),
                   lambda: eng.stream_rois_images((tensors[i] for i in idx), channels="RGB", **kw)):
            torch.cuda.synchronize()
            N.check(N.lib.ctpn_prof_enable(1), "ctpn_prof_enable")        # a run of its own: events bracket every launch
            list(fn())
            torch.cuda.synchronize()
            for e in N.prof_report():
                if e["kernel"] in ("resize_linear_u8_ragged", "resize_linear_u8_strided"):
                    got[e["kernel"]] = {"launches": e["launches"], "ms_per_batch": round(e["ms"] / max(1, e["launches"]), 5)}
            N.check(N.lib.ctpn_prof_enable(0), "ctpn_prof_enable")
        return got

    everything = list(range(n))
    subsets = {"%dx%d" % s: [i for i in everything if shapes[i] in (s, s[::-1])] for s in SIZES}
    rec["all"] = compare(everything)
    rec["per_source_size"] = {k: dict(images=len(idx), **compare(idx)) for k, idx in subsets.items()}
    # separate runs after the timed rounds: profiler census of the H2D bytes, then the library's kernel timings
    rec["h2d_bytes_per_image_census"] = {k: round(census_h2d(lambda: legs[k](everything)) / n) for k in legs}
    for k, idx in subsets.items():
        rec["per_source_size"][k]["h2d_bytes_per_image_census"] = {
            leg: round(census_h2d(lambda: legs[leg](idx)) / len(idx)) for leg in legs}
    rec["kernels"] = kernels(everything)
    for k, idx in subsets.items():
        rec["per_source_size"][k]["kernels"] = kernels(idx)
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
