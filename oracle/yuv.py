"""Oracle (test infrastructure; never imported by the product): numpy restatement of cv2.cvtColor for the YUV 4:2:0 codes
COLOR_YUV2BGR_NV12 / _NV21 / _I420 / _YV12.  OpenCV (opencv-python, 4.13.0 in this image) converts all four with BT.601
limited-range coefficients in 20-bit fixed point and nearest chroma: chroma sample (y >> 1, x >> 1) serves luma sample
(y, x), and

    u = U - 128, v = V - 128, yy = max(Y - 16, 0) * CY
    B = sat_u8((yy + HALF + CUB * u) >> 20)
    G = sat_u8((yy + HALF + CVG * v + CUG * u) >> 20)
    R = sat_u8((yy + HALF + CVR * v) >> 20)

with an arithmetic shift; every term fits in int32.  cv2 rejects odd widths and heights for these codes.  This is
cvtColor's conversion; cv2.VideoCapture's BGR frames come from FFmpeg's swscale, which rounds differently.  Pinned
against cv2.cvtColor in tests/test_yuv_frames_cpu.py (all 2^24 (Y, U, V) triples, and frames in all four layouts)."""
import numpy as np

CY, CUB, CUG, CVG, CVR = 1220542, 2116026, -409993, -852492, 1673527
SHIFT = 20
HALF = 1 << (SHIFT - 1)
LAYOUTS = ("NV12", "NV21", "I420", "YV12")


def yuv_to_bgr(Y, U, V):
    """Y [h, w], U and V [h/2, w/2] uint8 planes -> the BGR uint8 [h, w, 3] image cv2.cvtColor gives."""
    Y = np.asarray(Y).astype(np.int64)
    u = np.repeat(np.repeat(np.asarray(U).astype(np.int64), 2, 0), 2, 1) - 128
    v = np.repeat(np.repeat(np.asarray(V).astype(np.int64), 2, 0), 2, 1) - 128
    yy = np.maximum(Y - 16, 0) * CY + HALF
    b = (yy + CUB * u) >> SHIFT
    g = (yy + CVG * v + CUG * u) >> SHIFT
    r = (yy + CVR * v) >> SHIFT
    return np.clip(np.stack([b, g, r], -1), 0, 255).astype(np.uint8)


def planes_to_buffer(Y, U, V, layout):
    """The single [h*3/2, w] buffer cv2 reads for `layout` from Y, U, V planes."""
    h, w = Y.shape
    if layout in ("NV12", "NV21"):
        a, b = (U, V) if layout == "NV12" else (V, U)
        return np.concatenate([Y, np.stack([a, b], -1).reshape(h // 2, w)])
    a, b = (U, V) if layout == "I420" else (V, U)
    return np.concatenate([Y.ravel(), a.ravel(), b.ravel()]).reshape(h * 3 // 2, w)


def buffer_to_planes(buf, layout):
    """Y, U, V planes of a [h*3/2, w] buffer in cv2's `layout` (the inverse of planes_to_buffer)."""
    h, w = buf.shape[0] // 3 * 2, buf.shape[1]
    Y = buf[:h]
    if layout in ("NV12", "NV21"):
        a, b = buf[h:, 0::2], buf[h:, 1::2]
        return (Y, a, b) if layout == "NV12" else (Y, b, a)
    flat = buf[h:].ravel()
    a, b = flat[:h * w // 4].reshape(h // 2, w // 2), flat[h * w // 4:].reshape(h // 2, w // 2)
    return (Y, a, b) if layout == "I420" else (Y, b, a)
