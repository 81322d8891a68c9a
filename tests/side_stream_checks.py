#!/usr/bin/env python
"""F16F8 calibration of an Engine with streams > 1, run as a subprocess by tests/test_side_streams_gpu.py on the test library
(CTPN_B200_LIB=dbg, for ctpn_net_f16f8_scales).  Prints one JSON line {"ok": bool, ...} as its last line of stdout.

    calibration  a 32-image batch whose first 16 images are low-contrast, so that their activation maxima lie a binade or
                 more below those of the whole batch (asserted: an engine calibrated on the first 16 alone gets other
                 scales).  Engine(streams=2) must calibrate to Engine(streams=1)'s scales and return its results bit for
                 bit, on the first call and the next, after recalibrate() and after load_weights().

    CTPN_B200_LIB=dbg python tests/side_stream_checks.py calibration
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT, os.path.join(ROOT, "text-detection-ctpn_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def scales(eng):
    from ctpn_b200 import _native as N
    s, t, amax = ((C.c_float * 13)() for _ in range(3))
    N.check(N.lib.ctpn_net_f16f8_scales(eng._net, s, t, amax), "ctpn_net_f16f8_scales")
    return list(s), list(t), list(amax)


def low_contrast(im, gain):
    return np.clip(np.rint(128.0 + (im.astype(np.float64) - 128.0) * gain), 0, 255).astype(np.uint8)


def same_rois(a, b):
    return len(a) == len(b) and all(x.shape == y.shape and np.array_equal(x, y) for x, y in zip(a, b))


def cmd_calibration(a):
    import torch
    from ctpn_b200 import Engine
    from oracle import synth
    assert os.environ.get("CTPN_B200_LIB") == "dbg"
    w = synth.make_weights(0)
    ims = np.stack([synth.make_image(500 + i, a.H, a.W) for i in range(a.B)])
    ims[:a.B // 2] = low_contrast(ims[:a.B // 2], a.gain)
    half = Engine(w, mode="f16f8")
    half.forward_heads(torch.from_numpy(ims[:a.B // 2]).cuda())
    s_half = scales(half)
    del half
    one, two = Engine(w, mode="f16f8"), Engine(w, mode="f16f8", streams=2)
    res, ok = dict(steps=[]), True
    for step in ("first call", "second call", "recalibrate", "load_weights"):
        if step == "recalibrate":
            one.recalibrate()
            two.recalibrate()
        elif step == "load_weights":
            one.load_weights(w)
            two.load_weights(w)
        r1, r2 = one.rois_batch(ims), two.rois_batch(ims)
        s1, s2 = scales(one), scales(two)
        st = dict(step=step, scales_equal=s1[:2] == s2[:2], amax_equal=s1[2] == s2[2], rois_equal=same_rois(r1, r2),
                  t_one=s1[1], t_two=s2[1])
        res["steps"].append(st)
        ok = ok and st["scales_equal"] and st["amax_equal"] and st["rois_equal"]
    # the precondition: the first half alone calibrates to other scales than the whole batch
    differs = [l for l in range(13) if (s_half[0][l], s_half[1][l]) != (s1[0][l], s1[1][l])]
    res.update(half_t=s_half[1], half_differs_at=differs, precondition=bool(differs))
    ok = ok and bool(differs)
    res["ok"] = bool(ok)
    print(json.dumps(res))
    return 0 if ok else 1


def main(argv=None):
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    c = sub.add_parser("calibration")
    for k, d in dict(B=32, H=600, W=900).items():
        c.add_argument("--" + k, type=int, default=d)
    c.add_argument("--gain", type=float, default=0.25)
    a = ap.parse_args(argv)
    return {"calibration": cmd_calibration}[a.cmd](a)


if __name__ == "__main__":
    sys.exit(main())
