#!/usr/bin/env python
"""conv1_1 and conv1_2 at batch 32 x 1200x1600 (bench.py --config 4), run as a subprocess by tests/test_large_batches_gpu.py
so that a faulting kernel fails one test instead of the session.  Prints one JSON line {"ok": bool, ...} as its last line of
stdout, or {"ok": false, "skip": reason} when the device has too little free memory.

At this size one plane of conv1_1's output holds 32 * 1200 * 1600 * 64 = 3.93e9 elements (7.9 GB in bf16): element indices
pass 2^31, byte offsets pass 2^32 and the second plane's element indices pass 2^32.  `conv` runs ctpn_conv1_1_tc[_f16f8] on
random uint8 images and ctpn_conv3x3[_f16f8] 64 -> 64 with ReLU and the 2x2 pool on conv1_1's own output, and checks
  * every image's slice of both batch outputs bit for bit against the same kernel run on that image alone, and
  * sampled output pixels against float64 computed from the kernel's own inputs, with the bounds of tests/gpu_checks.py:
    the first and last pixel of every image, the pixels on both sides of every element index and byte offset 2^31 .. 2^35
    that falls inside an output (plane offset included), and for conv1_2 the pooled pixels that read those conv1_1 pixels.

    python tests/large_checks.py conv --mode bf16
    python tests/large_checks.py conv --mode f16f8
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

import gpu_checks  # noqa: E402
from gpu_checks import F_F32, F_POOL, F_RELU  # noqa: E402
from variant_checks import CONV1_TOL, CONV_TOL, _conv1_ref, _conv1_weights  # noqa: E402

P = 2                               # bf16 planes of the bf16x2 arithmetic (bench's other mode is F16F8)
F16F8_TOL, E4M3_REL = 6e-5, 0.07    # gpu_checks.cmd_conv_f16f8 / variant_checks.cmd_conv1_q: value + residual, e4m3 copy


def need_bytes(B, H, W):
    """Device memory of the check: images, conv1_1 output, conv1_2 output, one image's copies, float64 image-0 reference."""
    n1, n2 = B * H * W * 64, B * (H // 2) * (W // 2) * 64
    per_image = H * W * 64
    return B * H * W * 3 + 4 * n1 + 4 * n2 + 3 * 4 * per_image + 3 * 8 * per_image


def boundary_pixels(planes, npix, ks=range(31, 36)):
    """Pixels of an output next to element index / byte offset 2^k: planes is a list of (base byte, bytes per pixel, bytes
    per element) of the output's planes; for every k the pixels holding the bytes just below and at 2^k (byte offset) and
    at 2^k elements of that plane's element type counted from the tensor's start.  Returns sorted pixel numbers."""
    out = set()
    for base, bpp, esize in planes:
        for k in ks:
            for target in (1 << k, esize << k):
                for byte in (target - 1, target):
                    q = (byte - base) // bpp
                    if byte >= base and 0 <= q < npix:
                        out.add(int(q))
    return sorted(out)


def pix(q, H, W):
    return int(q // (H * W)), int(q // W % H), int(q % W)


def patch(t, b, y0, x0, n):
    """t[b, y0:y0+n, x0:x0+n] of a [B, H, W, ...] tensor as float64 numpy, zero outside the image (SAME padding)."""
    H, W = t.shape[1], t.shape[2]
    out = np.zeros((n, n) + tuple(t.shape[3:]), np.float64)
    ya, yb, xa, xb = max(y0, 0), min(y0 + n, H), max(x0, 0), min(x0 + n, W)
    out[ya - y0:yb - y0, xa - x0:xb - x0] = t[b, ya:yb, xa:xb].double().cpu().numpy()
    return out


def conv3x3_at(terms, bias):
    """float64 3x3 conv + ReLU + 2x2 max-pool at one pooled pixel: terms is a list of (zero-padded input patch [4, 4, Cin],
    weights [3, 3, Cin, Cout]) whose convolutions add up (one pair for bf16 planes, three for the F16F8 products) -> [Cout]."""
    ys = [np.maximum(sum(np.einsum("hwc,hwco->o", x[dy:dy + 3, dx:dx + 3], w) for x, w in terms) + bias, 0.0)
          for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1))]
    return np.max(ys, axis=0)


def cmd_conv(a):
    import torch
    from ctpn_b200 import _native as N
    from oracle import quant
    dev = torch.device("cuda", 0)
    B, H, W = a.B, a.H, a.W
    f8 = a.mode == "f16f8"
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info(dev)
    need = need_bytes(B, H, W)
    if free < need:
        print(json.dumps(dict(ok=False, skip="conv %s at %dx%dx%d needs %.1f GB of device memory, %.1f GB of %.1f GB are free"
                              % (a.mode, B, H, W, need / 1e9, free / 1e9, total / 1e9))))
        return 1
    rs = np.random.RandomState(a.seed)
    w1, b1, lut = _conv1_weights(rs)
    w2 = (rs.standard_normal((9, 64, 64)) * (2.0 / (9 * 64)) ** 0.5).astype(np.float32)
    b2 = (rs.standard_normal(64) * 0.1).astype(np.float32)
    w1d, b1d, lutd, w2d, b2d = (torch.from_numpy(x).to(dev) for x in (w1, b1, lut, w2, b2))
    g = torch.Generator(device=dev).manual_seed(a.seed)
    img = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8, device=dev, generator=g)
    Ho, Wo = H // 2, W // 2
    n1, n2 = B * H * W * 64, B * Ho * Wo * 64
    st = N.stream_ptr()

    # float64 conv1_1 of image 0: the output scale (and F16F8's out_t, as variant_checks.cmd_conv1_q picks it)
    x0 = torch.from_numpy(lut.astype(np.float64)).to(dev)[img[0].long(), torch.arange(3, device=dev)][None]
    scale1_0 = float(_conv1_ref(x0, w1, b1d).abs().max())
    del x0
    out_t1 = gpu_checks._pow2_floor(448.0 / scale1_0) / 2.0

    if f8:
        s_w, t_w = quant.weight_scales(float(np.abs(w2).max()))
        wp = torch.zeros(2 * 64 * 9 * 64 * 2, dtype=torch.uint8, device=dev)
        N.check(N.lib.ctpn_pack_weights_f16f8(N.ptr(w2d), 9, 64, 64, 64, s_w, t_w, N.ptr(wp), st), "pack f16f8")
        inv_main, inv_cross = 1.0 / s_w, 1.0 / (2048.0 * out_t1 * t_w)

        def conv1(src, nb, out):
            N.check(N.lib.ctpn_conv1_1_tc_f16f8(N.ptr(src), 0, N.ptr(lutd), N.ptr(w1d), N.ptr(b1d), N.ptr(out), nb, H, W, 1.0, out_t1, st),
                    "conv1_1_tc_f16f8")

        def conv2(src, nb, out, flags, out_t):
            N.check(N.lib.ctpn_conv3x3_f16f8(N.ptr(src), N.ptr(wp), N.ptr(b2d), N.ptr(out), nb, H, W, 64, 64, 9, flags, inv_main,
                                             inv_cross, 1.0, out_t, st), "conv3x3_f16f8")
        out1 = torch.empty(4 * n1, dtype=torch.uint8, device=dev)

        def image1(t, nb, b):          # image b of a flat F16F8 tensor, in the layout of a batch of one
            half = t.numel() // 2
            return torch.cat([t[:half].view(nb, -1)[b], t[half:].view(nb, -1)[b]])
    else:
        wp = torch.empty(P * 64 * 9 * 64, dtype=torch.bfloat16, device=dev)
        N.check(N.lib.ctpn_pack_weights(N.ptr(w2d), 9, 64, 64, 64, P, N.ptr(wp), st), "pack")

        def conv1(src, nb, out):
            N.check(N.lib.ctpn_conv1_1_tc(N.ptr(src), 0, N.ptr(lutd), N.ptr(w1d), N.ptr(b1d), N.ptr(out), nb, H, W, P, st), "conv1_1_tc")

        def conv2(src, nb, out, flags, out_t=None):
            N.check(N.lib.ctpn_conv3x3(N.ptr(src), N.ptr(wp), N.ptr(b2d), N.ptr(out), nb, H, W, 64, 64, 9, P, flags, st), "conv3x3")
        out1 = torch.empty((P, B, H, W, 64), dtype=torch.bfloat16, device=dev)

        def image1(t, nb, b):          # image b of a flat [P][B]... tensor, in the layout of a batch of one
            return t.view(P, nb, -1)[:, b].reshape(-1)

    # ---- the batch ----
    conv1(img, B, out1)
    flat1 = out1.view(-1)
    # conv1_2's output scale from image 0 alone, float32 output (F16F8's out_t)
    o32 = torch.empty((1, Ho, Wo, 64), dtype=torch.float32, device=dev)
    conv2(image1(flat1, B, 0).contiguous(), 1, o32, F_RELU | F_POOL | F_F32, 1.0)
    torch.cuda.synchronize()
    out_t2 = gpu_checks._pow2_floor(448.0 / max(float(o32.abs().max()), 1e-6)) / 2.0
    del o32
    out2 = torch.empty(4 * n2, dtype=torch.uint8, device=dev) if f8 else torch.empty((P, B, Ho, Wo, 64), dtype=torch.bfloat16, device=dev)
    conv2(out1, B, out2, F_RELU | F_POOL, out_t2)
    torch.cuda.synchronize()
    flat2 = out2.view(-1)

    # ---- every image alone, bit for bit ----
    bad_single, max1, max2 = [], 0.0, 0.0
    s1 = torch.empty(flat1.numel() // B, dtype=flat1.dtype, device=dev)
    s2 = torch.empty(flat2.numel() // B, dtype=flat2.dtype, device=dev)
    for b in range(B):
        conv1(img[b:b + 1].contiguous(), 1, s1)
        inp = image1(flat1, B, b).contiguous()
        conv2(inp, 1, s2, F_RELU | F_POOL, out_t2)
        e1, e2 = bool(torch.equal(s1, image1(flat1, B, b))), bool(torch.equal(s2, image1(flat2, B, b)))
        if not (e1 and e2):
            bad_single.append(dict(image=b, conv1_1=e1, conv1_2=e2))
        # output scales for the float64 bounds: max|value| over the batch (the fp16 plane, or the sum of the bf16 planes)
        if f8:
            max1 = max(max1, float(inp[:2 * H * W * 64].view(torch.float16).abs().max()))
            max2 = max(max2, float(s2[:2 * Ho * Wo * 64].view(torch.float16).abs().max()))
        else:
            max1 = max(max1, float(inp.view(P, -1).float().sum(0).abs().max()))
            max2 = max(max2, float(s2.view(P, -1).float().sum(0).abs().max()))
        del inp
    del s1, s2

    # ---- sampled pixels against float64 ----
    if f8:
        h1 = out1[:2 * n1].view(torch.float16).view(B, H, W, 64)
        c1 = out1[2 * n1:].view(B, H, W, 128)
        h2 = out2[:2 * n2].view(torch.float16).view(B, Ho, Wo, 64)
        c2 = out2[2 * n2:].view(B, Ho, Wo, 128)
        planes1, planes2 = [(0, 128, 2), (2 * n1, 128, 1)], [(0, 128, 2), (2 * n2, 128, 1)]
        wh_d, wv_d, wr_d = (t.numpy().reshape(64, 3, 3, 64).transpose(1, 2, 3, 0)
                            for t in quant.quantize(torch.from_numpy(w2).permute(2, 0, 1).contiguous(), s_w, t_w)[2])
    else:
        planes1 = [(p * 2 * n1, 128, 2) for p in range(P)]
        planes2 = [(p * 2 * n2, 128, 2) for p in range(P)]
        w2c = wp.view(P, 64, 9, 64).double().sum(0).cpu().numpy().reshape(64, 3, 3, 64).transpose(1, 2, 3, 0)   # HWIO, carried
    edge1 = boundary_pixels(planes1, B * H * W)
    edge2 = boundary_pixels(planes2, B * Ho * Wo)

    def first_last(h, w):
        return [(b, 0, 0) for b in range(B)] + [(b, h - 1, w - 1) for b in range(B)]
    px1 = sorted(set(first_last(H, W) + [pix(q, H, W) for q in edge1]))
    px2 = sorted(set(first_last(Ho, Wo) + [pix(q, Ho, Wo) for q in edge2] + [(b, y // 2, x // 2) for b, y, x in px1]))
    lut64 = lut.astype(np.float64)
    w1_64, b1_64, b2_64 = w1.astype(np.float64), b1.astype(np.float64), b2.astype(np.float64)

    def e4m3(u8):
        return torch.from_numpy(np.ascontiguousarray(u8, np.uint8)).view(torch.float8_e4m3fn).double().numpy()

    err1, err2, rel8_1, rel8_2 = 0.0, 0.0, 0.0, 0.0
    for b, y, x in px1:
        inside = np.zeros((3, 3, 1))
        inside[max(0, 1 - y):min(3, H + 1 - y), max(0, 1 - x):min(3, W + 1 - x)] = 1.0      # SAME padding of the mean-subtracted blob
        xin = lut64[patch(img, b, y - 1, x - 1, 3).astype(np.int64), np.arange(3)] * inside
        want = np.maximum(np.einsum("hwc,hwco->o", xin, w1_64) + b1_64, 0.0)
        if f8:
            hv = h1[b, y, x].double().cpu().numpy()
            cr = c1[b, y, x].cpu().numpy()
            got = hv + e4m3(cr[64:]) / (2048.0 * out_t1)
            rel8_1 = max(rel8_1, float((np.abs(e4m3(cr[:64]) / out_t1 - want) / (np.abs(want) + max1 * 2.0 ** -9)).max()))
        else:
            got = out1[:, b, y, x].double().sum(0).cpu().numpy()
        err1 = max(err1, float(np.abs(got - want).max()))
    for b, oy, ox in px2:
        if f8:
            hp = patch(h1, b, 2 * oy - 1, 2 * ox - 1, 4)
            cp = patch(c1, b, 2 * oy - 1, 2 * ox - 1, 4)
            va, ra = e4m3(cp[..., :64]) / out_t1, e4m3(cp[..., 64:]) / (2048.0 * out_t1)
            # y = h_a h_w + v_a r_w + r_a v_w (gpu_checks.cmd_conv_f16f8); a padded pixel is zero in all three parts
            want = conv3x3_at([(hp, wh_d), (va, wr_d), (ra, wv_d)], b2_64)
            hv = h2[b, oy, ox].double().cpu().numpy()
            cr = c2[b, oy, ox].cpu().numpy()
            got = hv + e4m3(cr[64:]) / (2048.0 * out_t2)
            rel8_2 = max(rel8_2, float((np.abs(e4m3(cr[:64]) / out_t2 - want) / (np.abs(want) + max2 * 2.0 ** -9)).max()))
        else:
            xp = sum(patch(out1[p], b, 2 * oy - 1, 2 * ox - 1, 4) for p in range(P))
            want = conv3x3_at([(xp, w2c)], b2_64)
            got = out2[:, b, oy, ox].double().sum(0).cpu().numpy()
        err2 = max(err2, float(np.abs(got - want).max()))
    tol1 = F16F8_TOL if f8 else CONV1_TOL[P]
    tol2 = F16F8_TOL if f8 else CONV_TOL[P]
    ok_f64 = err1 <= tol1 * max1 and err2 <= tol2 * max2 and (not f8 or (rel8_1 <= E4M3_REL and rel8_2 <= E4M3_REL))
    ok = not bad_single and ok_f64
    print(json.dumps(dict(ok=bool(ok), mode=a.mode, shape=[B, H, W], single_image_mismatches=bad_single, f64=bool(ok_f64),
                          conv1_1=dict(max_err=err1, scale=max1, rel=err1 / max(max1, 1e-30), tol=tol1, e4m3_rel=rel8_1),
                          conv1_2=dict(max_err=err2, scale=max2, rel=err2 / max(max2, 1e-30), tol=tol2, e4m3_rel=rel8_2),
                          sampled=[len(px1), len(px2)], boundary_pixels=[pix(q, H, W) for q in edge1],
                          conv1_1_bytes=int(flat1.numel() * flat1.element_size()), peak_gb=torch.cuda.max_memory_allocated() / 1e9)))
    return 0 if ok else 1


def main(argv=None):
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    c = sub.add_parser("conv")
    for k, d in dict(B=32, H=1200, W=1600, seed=0).items():
        c.add_argument("--" + k, type=int, default=d)
    c.add_argument("--mode", choices=["bf16", "f16f8"], default="bf16")
    a = ap.parse_args(argv)
    return {"conv": cmd_conv}[a.cmd](a)


if __name__ == "__main__":
    sys.exit(main())
