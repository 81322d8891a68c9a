"""YUV 4:2:0 test frames on the device, shared by tests/test_yuv_frames_gpu.py and tests/yuv_frames_cases.py (this file is
not collected by pytest: its name does not start with test_).  Every layout a video user hands over: cv2's four
single-buffer layouts, pitched surfaces, a luma surface padded to 16-row alignment with the chroma after the padding,
chroma in an allocation of its own, and even-offset crops of a larger frame.  Padding and the area around a crop hold
random bytes, so a read outside the frame changes the result."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT, os.path.join(ROOT, "text-detection-ctpn_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from oracle import yuv  # noqa: E402

LAYOUTS = ("NV12", "NV21", "I420", "YV12", "nv12_pitched", "i420_pitched", "nv12_padded_surface", "nv12_split", "crop")


def planes_of(bgr):
    """Y, U, V planes of a BGR image with even sides, as cv2.cvtColor(COLOR_BGR2YUV_I420) makes them."""
    import cv2
    return yuv.buffer_to_planes(cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420), "I420")


def random_planes(seed, h, w):
    rng = np.random.default_rng(seed)
    return (rng.integers(0, 256, (h, w), dtype=np.uint8), rng.integers(0, 256, (h // 2, w // 2), dtype=np.uint8),
            rng.integers(0, 256, (h // 2, w // 2), dtype=np.uint8))


def pitch_for(w):
    return 2048 if w <= 2048 else (w + 511) // 512 * 512


def device_frame(Y, U, V, layout, seed=0):
    """A YUV420 frame on the device holding the planes Y, U, V in `layout` (LAYOUTS)."""
    import torch
    from ctpn_b200 import YUV420
    h, w = Y.shape
    gen = torch.Generator(device="cuda").manual_seed(seed)

    def garbage(*shape):
        return torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda", generator=gen)

    if layout in yuv.LAYOUTS:
        return YUV420.from_buffer(torch.from_numpy(yuv.planes_to_buffer(Y, U, V, layout)).cuda(), layout)
    if layout in ("nv12_pitched", "i420_pitched"):
        P = pitch_for(w)
        buf = garbage(h * 3 // 2, P)
        buf[:h, :w] = torch.from_numpy(Y).cuda()
        if layout == "nv12_pitched":
            buf[h:, :w] = torch.from_numpy(np.stack([U, V], -1).reshape(h // 2, w)).cuda()
            return YUV420.from_buffer(buf[:, :w], "NV12")
        chroma = buf[h:].reshape(h, P // 2)                 # chroma rows at half the luma pitch: U rows, then V rows
        chroma[:, :w // 2] = torch.from_numpy(np.concatenate([U, V])).cuda()
        return YUV420.from_buffer(buf[:, :w], "I420")
    if layout == "nv12_padded_surface":                    # e.g. 1920 x 1088 luma for a 1080-row frame
        P, Hs = pitch_for(w), (h + 16) // 16 * 16
        surf = garbage(Hs + h // 2, P)
        surf[:h, :w] = torch.from_numpy(Y).cuda()
        surf[Hs:, :w] = torch.from_numpy(np.stack([U, V], -1).reshape(h // 2, w)).cuda()
        return YUV420.nv12(surf[:h, :w], surf[Hs:, :w])
    if layout == "nv12_split":
        return YUV420.nv12(torch.from_numpy(Y.copy()).cuda(), torch.from_numpy(np.stack([U, V], -1)).cuda())
    if layout == "crop":                                   # rows 4.., columns 6.. of a larger I420 frame
        big = YUV420.from_buffer(garbage((h + 8) * 3 // 2, w + 12), "I420")
        big.y[4:4 + h, 6:6 + w] = torch.from_numpy(Y).cuda()
        big.u[2:2 + h // 2, 3:3 + w // 2] = torch.from_numpy(U).cuda()
        big.v[2:2 + h // 2, 3:3 + w // 2] = torch.from_numpy(V).cuda()
        return YUV420(big.y[4:4 + h, 6:6 + w], big.u[2:2 + h // 2, 3:3 + w // 2], big.v[2:2 + h // 2, 3:3 + w // 2])
    raise ValueError(layout)


# video-like frame sizes (even sides): 720p, 1080p, 4K, portrait 1080p, and smaller even photos
VIDEO_SIZES = [(720, 1280), (1080, 1920), (2160, 3840), (1920, 1080), (480, 640), (1200, 1800), (300, 550), (38, 54)]


def video_photos(n=16):
    """n BGR images of VIDEO_SIZES (after a round trip through I420, so each is exactly what cv2.cvtColor gives for its
    frame) and their planes."""
    import cv2
    from oracle import synth
    out = []
    for i in range(n):
        h, w = VIDEO_SIZES[i % len(VIDEO_SIZES)]
        Y, U, V = planes_of(synth.make_image(1300 + i, h, w))
        bgr = cv2.cvtColor(yuv.planes_to_buffer(Y, U, V, "I420"), cv2.COLOR_YUV2BGR_I420)
        out.append((bgr, (Y, U, V)))
    return out


def frames_of(photos, layouts=LAYOUTS):
    """The photos' planes as device frames, layouts taken in turn."""
    return [device_frame(*p, layouts[i % len(layouts)], seed=i) for i, (_, p) in enumerate(photos)]
