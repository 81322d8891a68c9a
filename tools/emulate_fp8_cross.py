#!/usr/bin/env python
"""CPU emulation (design study for DESIGN.md §9, not product code): how much head accuracy does the fp32-faithful conv
mode lose if the two cross-plane terms a0*w1 + a1*w0 are computed with fp8 (e4m3) operands instead of bf16?

Every 3x3 layer is evaluated as  main + cross  with
  main  = conv(a0, w0)                                   a0 = bf16(a), w0 = bf16(w)         (exact products, f32/f64 sum)
  cross = conv(q(a0), q(w1)) + conv(q(a1), q(w0))        a1 = bf16(a - a0), w1 = bf16(w - w0)
where q() is bf16 (today's 3-MMA mode) or e4m3 with a per-tensor power-of-two scale (the proposed 2-unit mode:
e4m3 MMAs run at twice the bf16 rate).  The BiLSTM / FC / heads stay float32.  Compared against the float64
evaluation of the float32 model on one synthetic 600x900 image.

    python tools/emulate_fp8_cross.py [--height 600 --width 900 --seed 0]
"""
import argparse
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import net_cpu, synth  # noqa: E402


def bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


def e4m3(t):
    """Round to float8 e4m3 after scaling the tensor's max magnitude into [224, 448] by a power of two."""
    m = float(t.abs().max())
    if m == 0.0:
        return t
    s = 2.0 ** np.floor(np.log2(448.0 / m))
    return (t * s).to(torch.float32).to(torch.float8_e4m3fn).to(t.dtype) / s


def f16(t):
    return t.to(torch.float16).to(t.dtype)


def e4m3_head(t, headroom=3):
    """e4m3 with a static-style scale: the tensor's max lands `headroom` binades below 448 (calibrated scale + margin)."""
    m = float(t.abs().max())
    if m == 0.0:
        return t
    s = 2.0 ** (np.floor(np.log2(448.0 / m)) - headroom)
    return (t * s).to(torch.float32).to(torch.float8_e4m3fn).to(t.dtype) / s


def conv_stack(blob, weights, mode, acc=torch.float64):
    x = torch.from_numpy(np.ascontiguousarray(blob)).to(acc).permute(0, 3, 1, 2)
    for name, cin, cout, pool in net_cpu.CONV_LAYERS:
        w = torch.from_numpy(np.ascontiguousarray(weights[name + "/weights"])).to(acc).permute(3, 2, 0, 1)
        b = torch.from_numpy(weights[name + "/biases"]).to(acc)
        if mode == "exact":
            y = F.conv2d(x, w, b, padding=1)
        elif mode.startswith("f16"):
            # fp16 hi planes (11 significant bits, residual 2^-12) + e4m3 cross terms: 1 + 2 * 1/2 = 2 units
            a0 = f16(x.float()).to(acc)
            w0 = f16(w.float()).to(acc)
            y = F.conv2d(a0, w0, b, padding=1)
            if mode != "f16x1":
                a1 = (x - a0).float().to(acc)
                w1 = (w - w0).float().to(acc)
                if mode == "f16f8_25":       # 2.5 units: a * r_w exactly on fp16 operands (1 unit), r_a * w on e4m3 copies (1/2 unit)
                    y = y + F.conv2d(a0, f16(w1.float()).to(acc), None, padding=1) + F.conv2d(e4m3_head(a1), e4m3_head(w0), None, padding=1)
                else:
                    q = {"f16f8": e4m3, "f16f8h": e4m3_head, "f16x2": lambda t: f16(t.float()).to(acc)}[mode]
                    y = y + F.conv2d(q(a0), q(w1), None, padding=1) + F.conv2d(q(a1), q(w0), None, padding=1)
        else:
            a0 = bf16(x.float()).to(acc)
            w0 = bf16(w.float()).to(acc)
            y = F.conv2d(a0, w0, b, padding=1)
            if mode != "bf16x1":
                a1 = bf16((x - a0).float()).to(acc)
                w1 = bf16((w - w0).float()).to(acc)
                q = e4m3 if mode == "fp8cross" else (lambda t: t)
                y = y + F.conv2d(q(a0), q(w1), None, padding=1) + F.conv2d(q(a1), q(w0), None, padding=1)
        x = F.relu(y).float().to(acc)          # activations are stored as float32-equivalent planes
        if pool:
            x = F.max_pool2d(x, 2, 2)
    return x


def heads(feat, weights):
    N, C, H, W = feat.shape
    dt = torch.float64
    seq = feat.permute(0, 2, 3, 1).reshape(N * H, W, C).to(dt)
    t = lambda k: torch.from_numpy(np.ascontiguousarray(weights[k])).to(dt)  # noqa: E731
    fw = net_cpu.lstm_dir(seq, t(net_cpu.LSTM_FW + "/kernel"), t(net_cpu.LSTM_FW + "/bias"), False)
    bw = net_cpu.lstm_dir(seq, t(net_cpu.LSTM_BW + "/kernel"), t(net_cpu.LSTM_BW + "/bias"), True)
    fc = torch.cat([fw, bw], -1).reshape(N * H * W, 256) @ t("lstm_o/weights") + t("lstm_o/biases")
    return (fc @ t("rpn_cls_score/weights") + t("rpn_cls_score/biases")).numpy(), (fc @ t("rpn_bbox_pred/weights") + t("rpn_bbox_pred/biases")).numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=600)
    ap.add_argument("--width", type=int, default=900)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--modes", default="bf16x1,bf16x2,fp8cross,f16x1,f16f8,f16f8h,f16f8_25,f16x2")
    a = ap.parse_args()
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    w = synth.make_weights(0)
    im = synth.make_image(a.seed, a.height, a.width).astype(np.float32) - net_cpu.PIXEL_MEANS.astype(np.float32)
    blob = im[None].astype(np.float32)
    with torch.no_grad():
        ref_feat = conv_stack(blob, w, "exact")
        ref = heads(ref_feat, w)
        print("reference: |cls| max %.3f  |bbox| max %.3f  feature max %.3f" % (np.abs(ref[0]).max(), np.abs(ref[1]).max(), float(ref_feat.max())))
        for mode in a.modes.split(","):
            feat = conv_stack(blob, w, mode)
            got = heads(feat, w)
            fe = float((feat - ref_feat).abs().max() / ref_feat.abs().max())
            print("%-9s feature rel err %.2e | cls max abs err %.2e | bbox max abs err %.2e" %
                  (mode, fe, np.abs(got[0] - ref[0]).max(), np.abs(got[1] - ref[1]).max()), flush=True)


if __name__ == "__main__":
    main()
