#!/usr/bin/env python
"""Hardware probe (run on the GPU box): can a wgmma A-operand descriptor address a SHIFTED view of a
swizzled shared-memory matrix (start row not a multiple of 8, arbitrary stride between 8-row groups)?
Prints one line per configuration; 'abs-ok' means the tensor core read row  row0 + (m//8)*stride + m%8
and column n for every (m, n), i.e. the swizzle is a function of the absolute shared-memory address."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "text-detection-ctpn_b200"))
os.environ["CTPN_B200_LIB"] = "dbg"      # the probes live in the test library
from ctpn_b200 import _native as N  # noqa: E402

dev = torch.device("cuda", 0)
rows = 256
a_row = torch.arange(rows, dtype=torch.float32).view(rows, 1).expand(rows, 64).contiguous().to(torch.bfloat16).to(dev)
a_col = torch.arange(64, dtype=torch.float32).view(1, 64).expand(rows, 64).contiguous().to(torch.bfloat16).to(dev)
ident = torch.eye(64, dtype=torch.float32).to(torch.bfloat16).to(dev)
out = torch.zeros(128, 64, dtype=torch.float32, device=dev)


def run(a, row0, stride, mode):
    out.zero_()
    N.check(N.lib.ctpn_probe_umma_view(N.ptr(a), N.ptr(ident), rows, row0, stride, mode, N.ptr(out), N.stream_ptr()), "probe")
    torch.cuda.synchronize()
    return out.cpu().numpy().copy()


for row0, stride, mode in [(0, 8, 0), (8, 8, 0), (1, 8, 0), (1, 8, 1), (3, 10, 0), (3, 10, 1), (11, 10, 0), (11, 10, 1),
                           (16, 10, 0), (16, 10, 1), (5, 16, 0), (5, 16, 1), (0, 10, 0), (2, 9, 0), (2, 9, 1)]:
    d_row, d_col = run(a_row, row0, stride, mode), run(a_col, row0, stride, mode)
    m = np.arange(128)
    want_row = (row0 + (m // 8) * stride + m % 8)[:, None] * np.ones((1, 64))
    want_col = np.ones((128, 1)) * np.arange(64)[None, :]
    ok = np.array_equal(d_row, want_row) and np.array_equal(d_col, want_col)
    line = "row0=%2d stride=%2d base_offset_mode=%d : %s" % (row0, stride, mode, "abs-ok" if ok else "MISMATCH")
    if not ok:
        line += "  rows(m=0..17,chunk0)=%s  rows(m=0..9,chunk7)=%s  cols(m=0,chunks)=%s cols(m=1,chunks)=%s" % (
            d_row[:18, 0].astype(int).tolist(), d_row[:10, 56].astype(int).tolist(), d_col[0, ::8].astype(int).tolist(), d_col[1, ::8].astype(int).tolist())
    print(line, flush=True)
