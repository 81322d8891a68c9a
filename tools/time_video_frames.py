"""YUV 4:2:0 video frames in device memory: the fused conversion against converting first.  Sets of 64 NV12 frames made from
the synthetic photos with cv2.cvtColor(COLOR_BGR2YUV_I420): 1280x720; 1920x1080 in a pitched (2048-byte) surface of 1088
luma rows with the chroma after the padding, as video decoders lay 1080p out; 3840x2160; 1080x1920 portrait; and the four
mixed.  f16f8, batches of up to 32, a window of 64.  Legs, alternating in one process, medians of the rounds:
  stream_frames   the frames through Engine.stream_rois_images (conversion fused into the resize);
  list_frames     the frames through Engine.rois_images;
  stream_bgr      BGR tensors converted before timing, through the stream (the bound without any conversion);
  stream_convert  the frames converted to BGR tensors inside the timed loop, lazily, by a cv2-exact torch integer
                  expression (torch_yuv_to_bgr: what a user has to write without the fused path), through the stream.
All four legs return the same rois bit for bit (asserted), and torch_yuv_to_bgr equals cv2.cvtColor on every frame.
Reported per set: images/s (median, min, max), host CPU ms per image (time.process_time, all threads), H2D bytes per
image from a torch.profiler census of one run per leg after the timed rounds, and the resize kernels' ms per batch
from the library's CUDA-event profile (the YUV kernel of stream_frames beside the strided kernel of stream_bgr).  The
card's name and power limit are read in the same run.

    python tools/time_video_frames.py --rounds 5 --out profiles/video_frames_h100.json
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

from time_frontend import card  # noqa: E402

LEGS = ("stream_frames", "list_frames", "stream_bgr", "stream_convert")
SETS = {"1280x720": [(720, 1280)], "1920x1080_pitched_1088": [(1080, 1920)], "3840x2160": [(2160, 3840)],
        "1080x1920_portrait": [(1920, 1080)], "mixed": [(720, 1280), (1080, 1920), (2160, 3840), (1920, 1080)]}


def torch_yuv_to_bgr(f):
    """cv2.cvtColor(COLOR_YUV2BGR_NV12 / _I420 ...) of a YUV420 frame in torch int32 arithmetic -> uint8 [H, W, 3]."""
    import torch
    from oracle.yuv import CUB, CUG, CVG, CVR, CY, HALF, SHIFT
    y = f.y.to(torch.int32)
    u = (f.u.to(torch.int32) - 128).repeat_interleave(2, 0).repeat_interleave(2, 1)
    v = (f.v.to(torch.int32) - 128).repeat_interleave(2, 0).repeat_interleave(2, 1)
    yy = (y - 16).clamp_min(0) * CY + HALF
    bgr = torch.stack([yy + CUB * u, yy + CVG * v + CUG * u, yy + CVR * v], -1) >> SHIFT
    return bgr.clamp(0, 255).to(torch.uint8)


def census_h2d(fn, warm):
    """Bytes of every host-to-device copy of one run of fn, from a torch.profiler trace.  warm() runs first inside the
    profile (the profiler can lose the first device records after it starts); only copies inside fn's span count."""
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
    return sum(int(e.get("args", {}).get("bytes", 0)) for e in events
               if e.get("cat") == "gpu_memcpy" and "HtoD" in e["name"] and t0 <= e.get("ts", -1) <= t1)


def nv12_frame(Y, U, V, padded):
    """The planes as an NV12 frame on the device: one dense [H*3/2, W] buffer, or (padded) a 2048-byte-pitch surface with
    luma rows padded to a multiple of 16 plus 16 and the chroma after them."""
    import torch
    from ctpn_b200 import YUV420
    from oracle import yuv
    h, w = Y.shape
    if not padded:
        return YUV420.from_buffer(torch.from_numpy(yuv.planes_to_buffer(Y, U, V, "NV12")).cuda(), "NV12")
    Hs, P = (h + 15) // 16 * 16 + (16 if h % 16 == 0 else 0), max(2048, (w + 511) // 512 * 512)
    surf = torch.zeros((Hs + h // 2, P), dtype=torch.uint8, device="cuda")
    surf[:h, :w] = torch.from_numpy(Y).cuda()
    surf[Hs:, :w] = torch.from_numpy(np.stack([U, V], -1).reshape(h // 2, w)).cuda()
    return YUV420.nv12(surf[:h, :w], surf[Hs:, :w])


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="f16f8")
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--window", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds per set (at least 3)")
    ap.add_argument("--out", default=None, help="write the JSON record here as well")
    a = ap.parse_args(argv)

    import cv2
    import torch
    from ctpn_b200 import Engine, _native as N
    from ctpn_b200.synthetic import make_image, make_weights
    from oracle import yuv
    assert a.rounds >= 3, "at least 3 rounds"
    eng = Engine(make_weights(0), mode=a.mode)            # raises without a GPU: there is nothing to time on a CPU
    rec = {"tool": "time_video_frames", "frames_per_set": a.frames, "max_batch": a.max_batch, "window": a.window,
           "mode": a.mode, "rounds": a.rounds, "card": card(), "device": torch.cuda.get_device_name(0)}
    kw = dict(max_batch=a.max_batch, window=a.window)
    eng.rois_images([make_image(i, 600, 900) for i in range(8)], max_batch=8)      # F16F8 calibrates on real-sized images

    def make_set(sizes, padded):
        frames, bgr = [], []
        distinct = {}
        for i in range(a.frames):
            h, w = sizes[i % len(sizes)]
            key = (h, w, (i // len(sizes)) % 8)                # 8 distinct photos per size, each frame its own copy
            if key not in distinct:
                Y, U, V = yuv.buffer_to_planes(cv2.cvtColor(make_image(len(distinct), h, w), cv2.COLOR_BGR2YUV_I420), "I420")
                distinct[key] = (Y, U, V, cv2.cvtColor(yuv.planes_to_buffer(Y, U, V, "NV12"), cv2.COLOR_YUV2BGR_NV12))
            Y, U, V, ref = distinct[key]
            f = nv12_frame(Y, U, V, padded and (h, w) == (1080, 1920))
            assert np.array_equal(torch_yuv_to_bgr(f).cpu().numpy(), ref)          # the user's conversion is cv2's
            frames.append(f)
            bgr.append(torch.from_numpy(ref).cuda())
        return frames, bgr

    def kernels(frames, bgr):
        got = {}
        for fn in (lambda: eng.stream_rois_images(iter(frames), **kw), lambda: eng.stream_rois_images(iter(bgr), **kw)):
            torch.cuda.synchronize()
            N.check(N.lib.ctpn_prof_enable(1), "ctpn_prof_enable")        # a run of its own: events bracket every launch
            list(fn())
            torch.cuda.synchronize()
            for e in N.prof_report():
                if e["kernel"] in ("resize_linear_u8_yuv420", "resize_linear_u8_strided"):
                    got[e["kernel"]] = {"launches": e["launches"], "ms_per_batch": round(e["ms"] / max(1, e["launches"]), 5)}
            N.check(N.lib.ctpn_prof_enable(0), "ctpn_prof_enable")
        return got

    rec["sets"] = {}
    for name, sizes in SETS.items():
        frames, bgr = make_set(sizes, padded=True)
        legs = {"stream_frames": lambda: [r[0] for r in eng.stream_rois_images(iter(frames), **kw)],
                "list_frames": lambda: [r[0] for r in eng.rois_images(frames, max_batch=a.max_batch)],
                "stream_bgr": lambda: [r[0] for r in eng.stream_rois_images(iter(bgr), **kw)],
                "stream_convert": lambda: [r[0] for r in eng.stream_rois_images((torch_yuv_to_bgr(f) for f in frames), **kw)]}
        assert tuple(legs) == LEGS
        ref = None
        for k, f in legs.items():          # warm-up: workspaces, slot buffers; every leg gives the same rois
            f()
            out = f()
            ref = out if ref is None else ref
            assert len(out) == len(ref) and all(np.array_equal(x, y) for x, y in zip(out, ref)), k
        wall, cpu = {k: [] for k in legs}, {k: [] for k in legs}
        order = list(legs)
        for r in range(a.rounds):
            for k in order[r % len(order):] + order[:r % len(order)]:
                torch.cuda.synchronize()
                t0, c0 = time.perf_counter(), time.process_time()
                legs[k]()
                torch.cuda.synchronize()
                wall[k].append(time.perf_counter() - t0)
                cpu[k].append(time.process_time() - c0)
        m = len(frames)
        out = {"frames": m}
        for k in legs:
            ips = [m / t for t in wall[k]]
            out[k] = {"images_per_s_median": round(float(np.median(ips)), 2), "min": round(float(min(ips)), 2),
                      "max": round(float(max(ips)), 2), "host_cpu_ms_per_image_median": round(1e3 * float(np.median(cpu[k])) / m, 3),
                      "h2d_bytes_per_image_census": round(census_h2d(legs[k], lambda: eng.rois_images(frames[:2])) / m, 1)}
        out["kernels"] = kernels(frames, bgr)
        rec["sets"][name] = out
        print(json.dumps({name: out}), flush=True)
        del frames, bgr, legs
        torch.cuda.empty_cache()
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
