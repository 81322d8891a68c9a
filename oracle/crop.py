"""Oracle (test infrastructure; never imported by the product): the line-crop recipe and a numpy restatement of the
cv2.warpAffine that defines it.  A text line is a row [x1,y1,x2,y2,x3,y3,x4,y4,score] of the connector's output in the
resize_im frame, corners TL, TR, BL, BR; its crop of height Hc (2 <= Hc <= 256) is

    len  = sqrt((x2-x1)*(x2-x1) + (y2-y1)*(y2-y1))        float64, in this order, no FMA
    ht   = sqrt((x3-x1)*(x3-x1) + (y3-y1)*(y3-y1))
    Wc   = max(2, rint(Hc * len / max(ht, 1.0)))          rint: round half to even
    Minv = [[(x2-x1)/(Wc-1), (x3-x1)/(Hc-1), x1],         dst (0,0) -> TL, (Wc-1,0) -> TR, (0,Hc-1) -> BL
            [(y2-y1)/(Wc-1), (y3-y1)/(Hc-1), y1]]
    crop = cv2.warpAffine(resized, Minv, (Wc, Hc), flags=INTER_LINEAR | WARP_INVERSE_MAP, borderMode=BORDER_REPLICATE)

BR is not used (the affine map of three points fixes it).  OpenCV (opencv-python, 4.13.0 in this image) computes the
uint8 warp in fixed point:

  * adelta[x] = cvRound(M0 * x * 1024), bdelta[x] = cvRound(M3 * x * 1024);
  * per row y: X0 = cvRound((M1 * y + M2) * 1024) + 16, Y0 = cvRound((M4 * y + M5) * 1024) + 16;
  * X = (X0 + adelta[x]) >> 5, Y = (Y0 + bdelta[x]) >> 5; taps (X >> 5, Y >> 5) saturated to int16, fractions
    fx = X & 31, fy = Y & 31;
  * the four taps (x0, x0 + 1) x (y0, y0 + 1) are each clamped to the image (BORDER_REPLICATE);
  * weights 32 (32-fx)(32-fy), 32 fx (32-fy), 32 (32-fx) fy, 32 fx fy -- cv2's float32 products of multiples of 1/32 are
    exact and sum to 32768, so its weight-sum correction never applies;
  * dst = (sum w * p + 16384) >> 15.
cvRound is round half to even.  Pinned against cv2.warpAffine, with IPP on and off, in tests/test_line_crops_cpu.py."""
import numpy as np


def crop_width(line, Hc):
    """Wc of one line (a sequence of at least 6 float64 values) at crop height Hc, as a Python int."""
    x1, y1, x2, y2, x3, y3 = (np.float64(v) for v in line[:6])
    length = np.sqrt((x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1))
    ht = np.sqrt((x3 - x1) * (x3 - x1) + (y3 - y1) * (y3 - y1))
    return max(2, int(np.rint(np.float64(Hc) * length / max(ht, np.float64(1.0)))))


def crop_widths(lines, Hc):
    """Wc of every row of lines [m, >= 6] -> int64 [m]."""
    return np.array([crop_width(ln, Hc) for ln in np.asarray(lines, np.float64)], np.int64)


def crop_matrix(line, Hc, Wc=None):
    """Minv (float64 [2, 3]) of one line: destination pixel -> source point."""
    x1, y1, x2, y2, x3, y3 = (np.float64(v) for v in line[:6])
    Wc = crop_width(line, Hc) if Wc is None else int(Wc)
    return np.array([[(x2 - x1) / np.float64(Wc - 1), (x3 - x1) / np.float64(Hc - 1), x1],
                     [(y2 - y1) / np.float64(Wc - 1), (y3 - y1) / np.float64(Hc - 1), y1]], np.float64)


def warp_affine_u8(im, M, Wc, Hc):
    """cv2.warpAffine(im, M, (Wc, Hc), flags=INTER_LINEAR | WARP_INVERSE_MAP, borderMode=BORDER_REPLICATE) of a uint8
    [h, w, C] image -> uint8 [Hc, Wc, C]."""
    im = np.asarray(im)
    h, w = im.shape[:2]
    M = np.asarray(M, np.float64)
    x = np.arange(Wc, dtype=np.float64)
    y = np.arange(Hc, dtype=np.float64)
    adelta = np.rint(M[0, 0] * x * 1024).astype(np.int64)
    bdelta = np.rint(M[1, 0] * x * 1024).astype(np.int64)
    X0 = np.rint((M[0, 1] * y + M[0, 2]) * 1024).astype(np.int64) + 16
    Y0 = np.rint((M[1, 1] * y + M[1, 2]) * 1024).astype(np.int64) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    sx = np.clip(X >> 5, -32768, 32767)
    sy = np.clip(Y >> 5, -32768, 32767)
    fx, fy = X & 31, Y & 31
    x0, x1 = np.clip(sx, 0, w - 1), np.clip(sx + 1, 0, w - 1)
    y0, y1 = np.clip(sy, 0, h - 1), np.clip(sy + 1, 0, h - 1)
    src = im.astype(np.int64)
    w00 = (32 * (32 - fx) * (32 - fy))[..., None]
    w01 = (32 * fx * (32 - fy))[..., None]
    w10 = (32 * (32 - fx) * fy)[..., None]
    w11 = (32 * fx * fy)[..., None]
    acc = src[y0, x0] * w00 + src[y0, x1] * w01 + src[y1, x0] * w10 + src[y1, x1] * w11
    return np.clip((acc + 16384) >> 15, 0, 255).astype(np.uint8)


def line_crop(im, line, Hc):
    """The crop of one line out of the resize_im output im (uint8 [h, w, 3]) at height Hc: uint8 [Hc, Wc, 3]."""
    Wc = crop_width(line, Hc)
    return warp_affine_u8(im, crop_matrix(line, Hc, Wc), Wc, Hc)


def line_crops(im, lines, Hc):
    """Every line's crop, padded as the device returns them: (uint8 [m, Hc, max Wc, 3] with zeros at and past each
    line's Wc, int64 widths [m])."""
    lines = np.asarray(lines, np.float64).reshape(-1, 9)
    widths = crop_widths(lines, Hc)
    out = np.zeros((len(lines), Hc, int(widths.max()) if len(lines) else 0, 3), np.uint8)
    for j, ln in enumerate(lines):
        out[j, :, :widths[j]] = line_crop(im, ln, Hc)
    return out, widths
