#!/usr/bin/env python
"""Generate tests/golden/reference_nms_keep.npz with the REFERENCE's own CUDA NMS (lib/utils/nms_kernel.cu `_nms`, built by
oracle/Makefile into oracle/_ref/libref_nms.so) on the seeded sorted boxes of tests/test_nms_gpu.py.  Needs a GPU:

    python tests/golden/make_golden_nms.py [OUT.npz]
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import postproc, synth  # noqa: E402

CASES = [(3000, 0.7, False), (6000, 0.7, True), (2000, 0.2, True)]


def case_key(n, thresh, ctpn_like):
    return "n%d_t%g_%s" % (n, thresh, "ctpn" if ctpn_like else "generic")


def sorted_dets(n, ctpn_like):
    dets = synth.make_boxes(77 + n % 5, n, ctpn_like=ctpn_like)
    return np.ascontiguousarray(dets[postproc.order_desc(dets[:, 4])])


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "reference_nms_keep.npz")
    ref = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libref_nms.so"))
    ref.ref_nms.restype = None
    ref.ref_nms.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int]
    res = {}
    for n, thresh, like in CASES:
        dets = sorted_dets(n, like)
        keep = np.zeros(n, np.int32)
        num = C.c_int(0)
        ref.ref_nms(keep.ctypes.data, C.byref(num), dets.ctypes.data, n, 5, np.float32(thresh), 0)
        res[case_key(n, thresh, like)] = keep[:num.value].copy()
    np.savez_compressed(out, **res)
    print("wrote", out, {k: len(v) for k, v in res.items()})


if __name__ == "__main__":
    main()
