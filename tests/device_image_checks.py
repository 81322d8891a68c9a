#!/usr/bin/env python
"""Checks of photos already in device memory that run in a process of their own, started by tests/test_device_images_gpu.py:
a torch.profiler session, or torchvision's nvJPEG, stays out of the test session's process.  A profiler session leaves
state behind in the process (later sessions there can come back without their kernel records), and the other GPU tests
that count kernels with the profiler must not depend on what ran before them.  Prints one JSON line {"ok": bool, ...} as
its last line of stdout.

    census  a torch.profiler census of a warm device-input stream (RGB planes, max_batch 4, window 8): per batch one H2D
            of at most the sizes / im_info tail, one strided resize kernel, no device-to-device copy, no torch copy kernel
            and no dense resize kernel, and no stream or device synchronise beyond the end of the stream.
    nvjpeg  photos encoded by cv2 (4:2:0 and 4:4:4) and decoded by torchvision's nvJPEG give, through rois_images and
            stream_rois_images, the results of the same calls on the decoded pixels copied to the host.
    demo DIR  ctpn/demo.py --batch 4 --device-frontend --gpu-decode, with and without --stream, on JPEGs and one PNG, writes
            the res_*.txt that --device-frontend writes on PNGs of the pixels nvJPEG decoded; files go under DIR.

    python tests/device_image_checks.py census
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT, os.path.join(ROOT, "text-detection-ctpn_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

# 16 photos: upscale, exact 1/2, float rescale, portrait, tiny, f = 1 and a strong downscale
PHOTO_SIZES = [(240, 400), (1200, 1800), (300, 550), (200, 600), (450, 300), (37, 53), (600, 900), (1700, 2300)]


def photos(n=16):
    from oracle import synth
    return [synth.make_image(900 + i, *PHOTO_SIZES[i % len(PHOTO_SIZES)]) for i in range(n)]


def on_device(im, layout):
    """A CUDA tensor holding the BGR image `im` in `layout`, and the channel order the call must be told."""
    import torch
    h, w = im.shape[:2]
    if layout == "hwc":
        return torch.from_numpy(im).cuda(), "BGR"
    if layout == "rgb":
        return torch.from_numpy(np.ascontiguousarray(im[:, :, ::-1])).cuda(), "RGB"
    if layout in ("crop", "rgb_crop"):         # inside a larger frame, with garbage around it
        frame = torch.randint(0, 256, (h + 9, w + 13, 3), dtype=torch.uint8, device="cuda")
        src = im if layout == "crop" else im[:, :, ::-1]
        frame[4:4 + h, 6:6 + w] = torch.from_numpy(np.ascontiguousarray(src)).cuda()
        return frame[4:4 + h, 6:6 + w], ("BGR" if layout == "crop" else "RGB")
    if layout in ("chw", "rgb_chw"):           # planar, as decoders return it
        src = im if layout == "chw" else im[:, :, ::-1]
        return torch.from_numpy(np.ascontiguousarray(src.transpose(2, 0, 1))).cuda().permute(1, 2, 0), \
            ("BGR" if layout == "chw" else "RGB")
    raise ValueError(layout)


BGR_LAYOUTS = ("hwc", "crop", "chw")
RGB_LAYOUTS = ("rgb", "rgb_crop", "rgb_chw")


def device_list(images, layouts):
    """The images as tensors, layouts taken in turn (all of one channel order)."""
    out = [on_device(im, layouts[i % len(layouts)]) for i, im in enumerate(images)]
    assert len({c for _, c in out}) == 1
    return [t for t, _ in out], out[0][1]


def same(a, b):
    """Whether two lists of result tuples are equal, arrays bit for bit."""
    if len(a) != len(b):
        return False
    for x, y in zip(a, b):
        if len(x) != len(y):
            return False
        for u, v in zip(x, y):
            if isinstance(u, np.ndarray):
                if not (u.dtype == v.dtype and u.shape == v.shape and np.array_equal(u, v)):
                    return False
            elif u != v:
                return False
    return True


def jpegs(n=6):
    """cv2-encoded JPEGs of blurred synthetic photos (something a JPEG can hold), 4:2:0 and 4:4:4 in turn."""
    import cv2
    from oracle import synth
    out = []
    for i in range(n):
        h, w = PHOTO_SIZES[(i * 3) % len(PHOTO_SIZES)]
        im = cv2.GaussianBlur(synth.make_image(980 + i, h, w), (0, 0), 2.0)
        params = [cv2.IMWRITE_JPEG_QUALITY, 90]
        if i % 2:
            params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444]
        ok, data = cv2.imencode(".jpg", im, params)
        assert ok
        out.append(data.tobytes())
    return out


def census():
    import tempfile
    import torch
    from torch.profiler import ProfilerActivity, profile, record_function
    from ctpn_b200 import Engine, frontend_plan, ragged_plan
    from oracle import synth
    ims = photos()
    eng = Engine(synth.make_weights(0), mode="f16f8")
    tensors, channels = device_list(ims, RGB_LAYOUTS)
    batches = 0
    for k in range(0, len(ims), 8):
        plan = frontend_plan(ims[k:k + 8])
        batches += len(ragged_plan([p.blob for p in plan], [p.dtype for p in plan], 4))

    def run(ts=tensors):
        return list(eng.stream_rois_images(iter(ts), max_batch=4, window=8, channels=channels))

    want = run()                        # warm: calibration, workspaces, slot buffers
    run()
    torch.cuda.synchronize()
    # a short run goes first inside the profile: the profiler can lose the first device records after it starts
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        run(tensors[:4])
        torch.cuda.synchronize()
        with record_function("device_stream_run"):
            got = run()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    span = next(e for e in events if e.get("name") == "device_stream_run" and e.get("cat") == "user_annotation")
    t0, t1 = span["ts"], span["ts"] + span["dur"]
    inside = [e for e in events if e.get("ph") == "X" and t0 <= e.get("ts", -1) <= t1]
    copies = [e for e in inside if e.get("cat") == "gpu_memcpy"]
    uploads = [int(e.get("args", {}).get("bytes", -1)) for e in copies if "HtoD" in e["name"]]
    kernels = [e["name"] for e in inside if e.get("cat") == "kernel"]
    calls = [e["name"] for e in inside if e.get("cat") == "cuda_runtime"]
    res = dict(batches=batches, same=same(got, want), uploads=uploads, dtod=sum("DtoD" in e["name"] for e in copies),
               strided=sum("resize_linear_u8_strided" in k for k in kernels),
               unwanted=sorted({k for k in kernels if "resize_linear_u8_ragged" in k or "copy_kernel" in k.lower()}),
               stream_syncs=calls.count("cudaStreamSynchronize"), device_syncs=calls.count("cudaDeviceSynchronize"))
    res["ok"] = bool(res["same"] and len(uploads) == batches and all(0 < b <= 28 * 4 for b in uploads) and res["dtod"] == 0
                     and res["strided"] == batches and not res["unwanted"] and res["stream_syncs"] <= 3
                     and res["device_syncs"] == 0)
    return res


def nvjpeg():
    import torch
    import torchvision
    from torchvision.io import ImageReadMode, decode_jpeg
    from ctpn_b200 import Engine
    from oracle import synth
    eng = Engine(synth.make_weights(0), mode="f16f8")
    data = [torch.frombuffer(bytearray(d), dtype=torch.uint8) for d in jpegs()]
    decoded = decode_jpeg(data, mode=ImageReadMode.RGB, device="cuda")
    hwc = [t.permute(1, 2, 0) for t in decoded]
    host = [t.cpu().numpy() for t in hwc]
    want = eng.rois_images(host, channels="RGB", return_resized=True)
    res = dict(torchvision=torchvision.__version__, decoded_on_device=all(t.is_cuda and t.shape[0] == 3 for t in decoded),
               list_call=same(eng.rois_images(hwc, channels="RGB", return_resized=True), want),
               stream=same(list(eng.stream_rois_images(iter(hwc), channels="RGB", return_resized=True, max_batch=2, window=3)),
                           want))
    res["ok"] = res["decoded_on_device"] and res["list_call"] and res["stream"]
    return res


def demo_files(top):
    import cv2
    import torch
    from torchvision.io import ImageReadMode, decode_jpeg
    from ctpn import demo
    from oracle import synth
    npz = os.path.join(top, "w.npz")
    np.savez(npz, **synth.make_weights(0))
    jpg_dir, png_dir = os.path.join(top, "jpg"), os.path.join(top, "png")
    os.makedirs(jpg_dir)
    os.makedirs(png_dir)
    for i, d in enumerate(jpegs(7)):
        with open(os.path.join(jpg_dir, "im_%d.jpg" % i), "wb") as f:
            f.write(d)
        t = decode_jpeg(torch.frombuffer(bytearray(d), dtype=torch.uint8), mode=ImageReadMode.RGB, device="cuda")
        cv2.imwrite(os.path.join(png_dir, "im_%d.png" % i), np.ascontiguousarray(t.permute(1, 2, 0).cpu().numpy()[:, :, ::-1]))
    extra = synth.make_image(999, 500, 380)
    cv2.imwrite(os.path.join(jpg_dir, "im_7.png"), extra)
    cv2.imwrite(os.path.join(png_dir, "im_7.png"), extra)
    out = {}
    for name, folder, flags in (("ref", png_dir, []), ("gpu", jpg_dir, ["--gpu-decode"]),
                                ("gpu_stream", jpg_dir, ["--gpu-decode", "--stream"])):
        demo.RESULTS_DIR = os.path.join(top, "results_" + name)
        demo.main(["--weights", npz, "--planes", "2", "--images", os.path.join(folder, "*"), "--batch", "4",
                   "--device-frontend"] + flags)
        out[name] = {}
        for p in sorted(os.listdir(demo.RESULTS_DIR)):
            if p.endswith(".txt"):
                with open(os.path.join(demo.RESULTS_DIR, p), "rb") as f:
                    out[name][p] = f.read()
    res = dict(files=len(out["ref"]), gpu=out["gpu"] == out["ref"], gpu_stream=out["gpu_stream"] == out["ref"])
    res["ok"] = res["files"] == 8 and res["gpu"] and res["gpu_stream"]
    return res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("check", choices=["census", "nvjpeg", "demo"])
    ap.add_argument("dir", nargs="?", default=None, help="demo: where the files go")
    a = ap.parse_args(argv)
    res = census() if a.check == "census" else nvjpeg() if a.check == "nvjpeg" else demo_files(a.dir)
    print(json.dumps(res))
    return 0 if res["ok"] else 1


if __name__ == "__main__":
    sys.exit(main())
