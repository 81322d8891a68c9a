"""GPU: the epilogue handoff of conv_tc_kernel.

At BN <= 128 the two MMA warpgroups hand each finished tile to a dedicated epilogue warpgroup through one staging buffer,
in 64-channel halves, and run the next tile's MMAs while it is converted and stored.  What that ordering could break: a
half read before it is written or overwritten before it is read (between the two halves of a tile, and between the last
half of a tile and the first half of the CTA's next tile), and the store-transpose blocks of the epilogue warps.  The
cases below run 1, 2 and many tiles per CTA (and fewer work units than SMs), BN 64 / 128 / 256, taps 9 and 1, pooling,
row-stacked input and output, float32, F16F8 and bf16x2 outputs, 2-CTA multicast pairs with an odd tile count and ragged
batches.  Each is held to the float64 bounds of tests/variant_checks.py, to itself across two runs and, where a batch
can be split, to its single images, bit for bit."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RELU, POOL, F32, OUT_BF16X2 = 1, 2, 4, 8


def run_script(*args, timeout=600):
    cmd = [sys.executable, os.path.join(HERE, "variant_checks.py")] + [str(a) for a in args]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout)
    lines = [l for l in p.stdout.strip().splitlines() if l.startswith("{")]
    assert lines, "no result line.\nstdout:\n%s\nstderr:\n%s" % (p.stdout[-2000:], p.stderr[-3000:])
    res = json.loads(lines[-1])
    print(" ".join(str(a) for a in args), "->", json.dumps(res))
    assert res["ok"] and p.returncode == 0, "%s\nstderr:\n%s" % (json.dumps(res), p.stderr[-2000:])
    return res


def conv(B, H, W, cin, cout, taps, planes, flags):
    return ("conv", "--B", B, "--H", H, "--W", W, "--cin", cin, "--cout", cout, "--taps", taps, "--planes", planes, "--flags", flags)


def f16f8(B, H, W, cin, cout, taps, flags, xscale=1.0):
    return ("conv_f16f8", "--B", B, "--H", H, "--W", W, "--cin", cin, "--cout", cout, "--taps", taps, "--flags", flags,
            "--xscale", xscale)


# A 3x3 layer runs on one CTA per SM once it has at least 16 output tiles per SM (132 SMs: 2112 tiles), else on 2-CTA
# clusters; the comments give the tiles (or cluster units) per CTA on a 132-SM H100.
FLOAT64_CASES = {
    "f16f8_bn128_many": f16f8(1, 300, 450, 64, 256, 9, RELU),                  # 2166 tiles: 16-17 per CTA, two halves each
    "f16f8_bn64_many_pool": f16f8(2, 300, 450, 64, 64, 9, RELU | POOL, 4.0),   # 2166 tiles of one half, pooled
    "f16f8_bn128_mc_odd": f16f8(1, 40, 72, 128, 256, 9, RELU),                 # 27 pixel tiles: odd pair count, 1 unit per CTA
    "f16f8_bn128_mc_two": f16f8(1, 150, 225, 64, 128, 9, RELU | POOL),         # 290 tiles: 1-2 units per cluster
    "f16f8_t1_bn128_many": f16f8(1, 1, 66304, 64, 512, 1, 0),                  # FC-shaped GEMM of a 32-image batch: 2072 tiles
    "f16f8_t1_bn64_two": f16f8(1, 1, 264 * 128, 64, 64, 1, 0),                 # exactly 2 tiles per CTA
    "bf16x2_bn128_many": conv(1, 300, 450, 64, 256, 9, 2, RELU),               # bf16-plane stores through the 512-B blocks
    "bf16x3_bn128_many_pool": conv(1, 300, 450, 64, 256, 9, 3, RELU | POOL),
    "bf16_bn256_many": conv(1, 300, 450, 64, 512, 9, 1, RELU),                 # BN = 256: the in-warpgroup epilogue
    "bf16x2_bn64_f32": conv(2, 300, 450, 64, 64, 9, 2, RELU | F32),            # float32 output, 2166 tiles
    "bf16x2_t1_bn128_f32": conv(1, 1, 66304, 64, 1024, 1, 2, F32),             # x-projection-shaped GEMM: 4144 tiles
}


@pytest.mark.parametrize("case", list(FLOAT64_CASES))
def test_handoff_against_float64(case):
    run_script(*FLOAT64_CASES[case])


@pytest.mark.parametrize("B,planes,promote", [(12, 2, 0), (5, 3, 0), (3, 1, 0)])
def test_row_stacked_planes_many_tiles(B, planes, promote):
    """Row-stacked input and output (conv5-shaped) at batches with several tiles per CTA equal the plain layout."""
    run_script("stack_planes", "--B", B, "--H", 37, "--W", 56, "--cin", 512, "--cout", 512, "--planes", planes,
               "--promote", promote)


# ---- run-to-run and batch-to-single-image equality, bit for bit ----------------------------------------------------------

def _native():
    sys.path.insert(0, os.path.join(ROOT, "text-detection-ctpn_b200"))
    import torch
    from ctpn_b200 import _native as N
    return torch, N


LAYERS = [   # (B, H, W, Cin, Cout, taps, flags): single-CTA and multicast 3x3 layers, pooled and not, and a GEMM
    (4, 150, 225, 128, 256, 9, RELU),
    (2, 300, 450, 64, 64, 9, RELU | POOL),
    (3, 40, 72, 256, 256, 9, RELU | POOL),
    (1, 1, 66304, 256, 512, 1, 0),
]


@pytest.mark.parametrize("mode", ["f16f8", "f16f8_f32", "f16f8_bf16x2", "bf16x2", "bf16", "bf16x2_f32"])
@pytest.mark.parametrize("layer", range(len(LAYERS)), ids=lambda i: "B%d_%dx%d_c%d-%d_t%d_f%d" % LAYERS[i])
def test_repeat_and_single_images_bit_identical(layer, mode):
    torch, N = _native()
    B, H, W, cin, cout, taps, flags = LAYERS[layer]
    f8 = mode.startswith("f16f8")
    planes = 1 if mode == "bf16" else 2
    if mode.endswith("_f32"):
        flags |= F32
    if mode == "f16f8_bf16x2":
        flags |= OUT_BF16X2
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(layer)
    # operands: bf16 / fp16 + e4m3 bit patterns of small magnitude (the exponent bits are capped), per plane [P][B][H][W][C]
    x = (torch.randint(0, 1 << 14, (planes, B, H, W, cin), dtype=torch.int32, device=dev, generator=g) & 0x3dff).to(torch.int16)
    w = (torch.randint(0, 1 << 14, (planes, cout, taps * cin), dtype=torch.int32, device=dev, generator=g) & 0x3dff).to(torch.int16)
    if f8:   # plane 1 holds e4m3 bytes: keep them finite (no 0x7f / 0xff)
        x[1] &= 0x3d3d
        w[1] &= 0x3d3d
    bias = torch.randn(cout, dtype=torch.float32, device=dev, generator=g)
    pool = bool(flags & POOL)
    ho, wo = (H // 2, W // 2) if pool else (H, W)
    oplanes = 1 if flags & F32 else planes
    oelem = 4 if flags & F32 else 2

    def run(xx, nb):
        out = torch.zeros(oplanes * nb * ho * wo * cout * oelem, dtype=torch.uint8, device=dev)
        if f8:
            N.check(N.lib.ctpn_conv3x3_f16f8(N.ptr(xx), N.ptr(w), N.ptr(bias), N.ptr(out), nb, H, W, cin, cout, taps, flags,
                                             0.5, 0.25, 0.75, 2.0, N.stream_ptr()), "conv")
        else:
            N.check(N.lib.ctpn_conv3x3(N.ptr(xx), N.ptr(w), N.ptr(bias), N.ptr(out), nb, H, W, cin, cout, taps, planes, flags,
                                       N.stream_ptr()), "conv")
        torch.cuda.synchronize()
        return out.view(oplanes, nb, -1)

    a = run(x, B)
    assert torch.equal(a, run(x, B)), "two runs differ"
    if B > 1:
        for b in (0, B - 1):
            one = run(x[:, b:b + 1].contiguous(), 1)
            assert torch.equal(one[:, 0], a[:, b]), "image %d alone differs from the batch" % b


@pytest.mark.parametrize("mode", ["f16f8", "bf16x2", "bf16"])
def test_ragged_batch_equals_single_images(mode):
    """A ragged batch (per-image extents: the epilogue's live mask) equals each image run alone at its own size."""
    import torch
    sys.path.insert(0, os.path.join(ROOT, "text-detection-ctpn_b200"))
    sys.path.insert(0, ROOT)
    from ctpn_b200 import Engine
    from oracle import synth
    eng = Engine(synth.make_weights(0), mode=mode)
    ims = np.stack([synth.make_image(200 + i, 600, 900) for i in range(3)])
    sizes = np.array([[600, 900], [480, 700], [352, 544]], np.int32)
    x = torch.from_numpy(ims).cuda()
    cls_b, box_b = eng.forward_heads(x, sizes=sizes)   # f16f8: the first call calibrates the activation scales
    cls_2, box_2 = eng.forward_heads(x, sizes=sizes)
    assert torch.equal(cls_b, cls_2) and torch.equal(box_b, box_2)
    for i, (h, w) in enumerate(sizes):
        c1, b1 = eng.forward_heads(torch.from_numpy(np.ascontiguousarray(ims[i:i + 1, :h, :w])).cuda())
        fh, fw = c1.shape[1], c1.shape[2]
        assert torch.equal(c1[0], cls_b[i, :fh, :fw]) and torch.equal(b1[0], box_b[i, :fh, :fw]), i
