#!/usr/bin/env python
"""Stand-alone GPU checks, run as subprocesses by the -m gpu tests so that a faulting kernel
(device trap, launch failure) cannot poison the pytest process.  Each sub-command prints one
JSON line {"ok": bool, ...} as its last line of stdout.

    python tests/gpu_checks.py conv --B 2 --H 37 --W 56 --cin 128 --cout 128 --taps 9 --planes 2 --flags 1
    python tests/gpu_checks.py bilstm --R 37 --W 56 --planes 2
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "text-detection-ctpn_b200"))

F_RELU, F_POOL, F_F32 = 1, 2, 4


def split_planes_t(x, planes):
    """float32 tensor -> [P, ...] bf16 planes with x ~= sum(planes) (same rule as the kernels)."""
    import torch
    out, r = [], x.clone()
    for _ in range(planes):
        h = r.to(torch.bfloat16)
        out.append(h)
        r = r - h.to(torch.float32)
    return torch.stack(out, 0)


def cmd_conv(a):
    import torch
    from ctpn_b200 import _native as N
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda", 0)
    g = torch.Generator(device="cpu").manual_seed(a.seed)
    x = torch.randn(a.B, a.H, a.W, a.cin, generator=g)
    x = torch.relu(x) if a.nonneg else x
    w = torch.randn(a.taps, a.cin, a.cout, generator=g) * (2.0 / (a.taps * a.cin)) ** 0.5
    b = torch.randn(a.cout, generator=g) * 0.1
    xp = split_planes_t(x.to(dev), a.planes).contiguous()                       # [P,B,H,W,C]
    wp_dev = torch.empty(a.planes * a.cout * a.taps * a.cin, dtype=torch.bfloat16, device=dev)
    w_dev, b_dev = w.to(dev).contiguous(), b.to(dev).contiguous()
    N.check(N.lib.ctpn_pack_weights(N.ptr(w_dev), a.taps, a.cin, a.cout, a.cout, a.planes, N.ptr(wp_dev), N.stream_ptr()), "pack")
    pool = bool(a.flags & F_POOL)
    Ho, Wo = (a.H // 2, a.W // 2) if pool else (a.H, a.W)
    if a.flags & F_F32:
        out = torch.full((a.B, Ho, Wo, a.cout), float("nan"), dtype=torch.float32, device=dev)
    else:
        out = torch.zeros((a.planes, a.B, Ho, Wo, a.cout), dtype=torch.bfloat16, device=dev)
    fn = N.lib.ctpn_conv3x3_simt if a.impl == "simt" else N.lib.ctpn_conv3x3
    N.check(fn(N.ptr(xp), N.ptr(wp_dev), N.ptr(b_dev), N.ptr(out), a.B, a.H, a.W, a.cin, a.cout, a.taps, a.planes,
               a.flags, N.stream_ptr()), "conv")
    torch.cuda.synchronize()
    got = out.double() if a.flags & F_F32 else out.double().sum(0)
    # reference: float64 conv on the exact values the planes carry
    xr = xp.double().sum(0).permute(0, 3, 1, 2)
    wr = wp_dev.view(a.planes, a.cout, a.taps, a.cin).double().sum(0)          # [Cout, taps, Cin]
    k = 3 if a.taps == 9 else 1
    wr = wr.view(a.cout, k, k, a.cin).permute(0, 3, 1, 2)
    y = torch.nn.functional.conv2d(xr, wr, b_dev.double(), padding=k // 2)
    if a.flags & F_RELU:
        y = torch.relu(y)
    if pool:
        y = torch.nn.functional.max_pool2d(y, 2, 2)
    y = y.permute(0, 2, 3, 1)
    err = (got - y).abs()
    scale = y.abs().max().item()
    max_err = err.max().item()
    nan = int(torch.isnan(got).sum().item())
    # bounds: P=1 output rounding to bf16 (2^-9); P>=2 the tensor core's truncating float32 accumulation (~K/16 * 2^-24)
    tol = {1: 6e-3, 2: 4e-5, 3: 2e-5}[a.planes] if not (a.flags & F_F32) else {1: 2e-5, 2: 2e-5, 3: 2e-5}[a.planes]
    ok = nan == 0 and max_err <= tol * max(scale, 1e-6)
    res = dict(ok=bool(ok), max_err=max_err, scale=scale, rel=max_err / max(scale, 1e-30), tol=tol, nan=nan)
    if not ok:
        idx = torch.nonzero(err > tol * scale)[:8].tolist()
        res["first_bad"] = idx
        res["bad_frac"] = float((err > tol * scale).double().mean().item())
        res["got"] = [got[tuple(i)].item() for i in idx]
        res["want"] = [y[tuple(i)].item() for i in idx]
    print(json.dumps(res))
    return 0 if ok else 1


def _pow2_floor(v):
    from oracle import quant
    return quant.pow2_floor(v)


def f16f8_quantize(x, s, t):
    """The F16F8 operand format (csrc/common.cuh) as restated on the CPU in oracle/quant.py."""
    from oracle import quant
    return quant.quantize(x, s, t)


def cmd_conv_f16f8(a):
    """ctpn_conv3x3_f16f8 against a float64 evaluation of exactly the operand values the planes carry:
    y = conv(h_a, h_w) + conv(q(a), q(r_w)) + conv(q(r_a), q(w)) (+bias, ReLU, pool), for float32, F16F8 and bf16x2 outputs;
    also checks the device weight packer bit for bit."""
    import torch
    from ctpn_b200 import _native as N
    dev = torch.device("cuda", 0)
    g = torch.Generator(device="cpu").manual_seed(a.seed)
    x = torch.relu(torch.randn(a.B, a.H, a.W, a.cin, generator=g)) * a.xscale
    w = torch.randn(a.taps, a.cin, a.cout, generator=g) * (2.0 / (a.taps * a.cin)) ** 0.5
    b = torch.randn(a.cout, generator=g) * 0.1
    s_in, t_in = 1.0, _pow2_floor(448.0 / float(x.abs().max())) / 2.0
    s_w, t_w = _pow2_floor(16384.0 / float(w.abs().max())), _pow2_floor(448.0 / float(w.abs().max()))
    xh, xc, (xh_d, xv_d, xr_d) = f16f8_quantize(x, s_in, t_in)
    inp = torch.cat([xh.view(torch.uint8).reshape(-1), xc.reshape(-1)]).to(dev)
    # weights: device packer vs the same rules in torch, on [Cout][taps][Cin]
    wt = w.permute(2, 0, 1).contiguous()
    wh, wc, (wh_d, wv_d, wr_d) = f16f8_quantize(wt, s_w, t_w)
    # weight cross rows are residual-first: swap the halves of every 128-byte block
    wc = torch.cat([wc[..., 64:], wc[..., :64]], dim=-1).contiguous()
    want_w = torch.cat([wh.view(torch.uint8).reshape(-1), wc.reshape(-1)])
    wp = torch.zeros(want_w.numel(), dtype=torch.uint8, device=dev)
    w_dev, b_dev = w.to(dev).contiguous(), b.to(dev).contiguous()
    N.check(N.lib.ctpn_pack_weights_f16f8(N.ptr(w_dev), a.taps, a.cin, a.cout, a.cout, s_w, t_w, N.ptr(wp), N.stream_ptr()), "pack")
    torch.cuda.synchronize()
    pack_ok = bool(torch.equal(wp.cpu(), want_w))
    # float64 reference on the carried values
    k = 3 if a.taps == 9 else 1

    def conv64(xd, wd):
        return torch.nn.functional.conv2d(xd.to(dev).permute(0, 3, 1, 2), wd.to(dev).view(a.cout, k, k, a.cin).permute(0, 3, 1, 2), None, padding=k // 2)
    y = conv64(xh_d, wh_d) + conv64(xv_d, wr_d) + conv64(xr_d, wv_d) + b_dev.double().view(1, -1, 1, 1)
    if a.flags & F_RELU:
        y = torch.relu(y)
    pool = bool(a.flags & F_POOL)
    if pool:
        y = torch.nn.functional.max_pool2d(y, 2, 2)
    y = y.permute(0, 2, 3, 1).contiguous()
    Ho, Wo = y.shape[1], y.shape[2]
    scale = y.abs().max().item()
    inv_main, inv_cross = 1.0 / (s_in * s_w), 1.0 / (2048.0 * t_in * t_w)
    out_s, out_t = 1.0, _pow2_floor(448.0 / max(scale, 1e-6)) / 2.0
    res = {"pack_ok": pack_ok}

    def run(flags, out):
        N.check(N.lib.ctpn_conv3x3_f16f8(N.ptr(inp), N.ptr(wp), N.ptr(b_dev), N.ptr(out), a.B, a.H, a.W, a.cin, a.cout, a.taps, flags,
                                         inv_main, inv_cross, out_s, out_t, N.stream_ptr()), "conv_f16f8")
        torch.cuda.synchronize()
    # (1) float32 output: only accumulation error
    o32 = torch.full((a.B, Ho, Wo, a.cout), float("nan"), dtype=torch.float32, device=dev)
    run(a.flags | F_F32, o32)
    e32 = (o32.double() - y).abs().max().item()
    res.update(f32_err=e32, scale=scale, f32_nan=int(torch.isnan(o32).sum().item()))
    # (2) F16F8 planes
    nel = a.B * Ho * Wo * a.cout
    oq = torch.zeros(nel * 4, dtype=torch.uint8, device=dev)
    run(a.flags, oq)
    h = oq[:nel * 2].view(torch.float16).double().view(a.B, Ho, Wo, a.cout)
    cr = oq[nel * 2:].view(a.B, Ho, Wo, a.cout // 64, 128)
    v8 = cr[..., :64].contiguous().view(torch.float8_e4m3fn).double().reshape(a.B, Ho, Wo, a.cout) / out_t
    r8 = cr[..., 64:].contiguous().view(torch.float8_e4m3fn).double().reshape(a.B, Ho, Wo, a.cout) / (2048.0 * out_t)
    eq_hr = ((h / out_s + r8) - y).abs().max().item()        # value + residual: ~2^-16 relative
    eq_v8 = ((v8 - y).abs() / (y.abs() + scale * 2.0 ** -9)).max().item()     # e4m3 copy: 2^-4 relative (+ subnormal floor)
    res.update(q_err_h_plus_r=eq_hr, q_rel_err_e4m3=eq_v8)
    # (3) two bf16 planes
    ob = torch.zeros((2, a.B, Ho, Wo, a.cout), dtype=torch.bfloat16, device=dev)
    run(a.flags | 8, ob)
    eb = (ob.double().sum(0) - y).abs().max().item()
    res.update(bf16x2_err=eb)
    ok = (pack_ok and res["f32_nan"] == 0 and e32 <= 2e-5 * scale and eq_hr <= 6e-5 * scale and eq_v8 <= 0.07 and eb <= 4e-5 * scale)
    res["ok"] = bool(ok)
    print(json.dumps(res))
    return 0 if ok else 1


def cmd_conv_stack(a):
    """Row-stacked batches (CTPN_F_STACK_IN / _OUT): the same layer on [B][H+1][W][C] frames with zero pad rows must give
    bit-identical image rows to the plain layout, zero pad rows in a stacked output, and compact rows otherwise."""
    import torch
    from ctpn_b200 import _native as N
    dev = torch.device("cuda", 0)
    g = torch.Generator(device="cpu").manual_seed(a.seed)
    B, H, W, C, Co = a.B, a.H, a.W, a.cin, a.cout
    x = torch.relu(torch.randn(B, H, W, C, generator=g))
    w = torch.randn(9, C, Co, generator=g) * (2.0 / (9 * C)) ** 0.5
    b = torch.randn(Co, generator=g) * 0.1
    s_in, t_in = 1.0, _pow2_floor(448.0 / float(x.abs().max())) / 2.0
    s_w, t_w = _pow2_floor(16384.0 / float(w.abs().max())), _pow2_floor(448.0 / float(w.abs().max()))
    xh, xc, _ = f16f8_quantize(x, s_in, t_in)
    plain = torch.cat([xh.view(torch.uint8).reshape(-1), xc.reshape(-1)]).to(dev)
    xs = torch.zeros(B, H + 1, W, C)
    xs[:, :H] = x
    sh, sc, _ = f16f8_quantize(xs, s_in, t_in)
    stacked = torch.cat([sh.view(torch.uint8).reshape(-1), sc.reshape(-1)]).to(dev)
    wp = torch.zeros(2 * Co * 9 * C * 2, dtype=torch.uint8, device=dev)
    N.check(N.lib.ctpn_pack_weights_f16f8(N.ptr(w.to(dev).contiguous()), 9, C, Co, Co, s_w, t_w, N.ptr(wp), N.stream_ptr()), "pack")
    bd = b.to(dev)
    inv_main, inv_cross, out_s, out_t = 1.0 / (s_in * s_w), 1.0 / (2048.0 * t_in * t_w), 1.0, 4.0

    def run(inp, flags, nbytes):
        out = torch.full((nbytes,), 0xAB, dtype=torch.uint8, device=dev)
        N.check(N.lib.ctpn_conv3x3_f16f8(N.ptr(inp), N.ptr(wp), N.ptr(bd), N.ptr(out), B, H, W, C, Co, 9, flags, inv_main, inv_cross,
                                         out_s, out_t, N.stream_ptr()), "conv")
        torch.cuda.synchronize()
        return out.cpu()
    n = B * H * W * Co
    ns = B * (H + 1) * W * Co
    ref = run(plain, F_RELU, 4 * n)                                     # plain in, plain F16F8 out
    so = run(stacked, F_RELU | 16 | 32, 4 * ns)                         # stacked in, stacked out
    co = run(stacked, F_RELU | 16, 4 * n)                               # stacked in, compact out
    cb = run(stacked, F_RELU | 16 | 8, 4 * n)                           # stacked in, compact bf16x2 out
    rb = run(plain, F_RELU | 8, 4 * n)
    ok_compact = bool(torch.equal(co, ref)) and bool(torch.equal(cb, rb))
    h_ref, c_ref = ref[:2 * n].view(B, H, W * Co * 2), ref[2 * n:].view(B, H, W * Co * 2)
    h_so, c_so = so[:2 * ns].view(B, H + 1, W * Co * 2), so[2 * ns:].view(B, H + 1, W * Co * 2)
    ok_rows = bool(torch.equal(h_so[:, :H], h_ref)) and bool(torch.equal(c_so[:, :H], c_ref))
    ok_pad = bool((h_so[:, H] == 0).all()) and bool((c_so[:, H] == 0).all())
    # pooled layer writing a stacked output: image rows equal the plain pooled output, pad rows untouched (0xAB here)
    pp = run(plain, F_RELU | F_POOL, 4 * B * (H // 2) * (W // 2) * Co)
    ps = run(plain, F_RELU | F_POOL | 32, 4 * B * (H // 2 + 1) * (W // 2) * Co)
    n2, n2s = B * (H // 2) * (W // 2) * Co, B * (H // 2 + 1) * (W // 2) * Co
    ok_pool = bool(torch.equal(ps[:2 * n2s].view(B, H // 2 + 1, -1)[:, :H // 2], pp[:2 * n2].view(B, H // 2, -1))) and \
        bool(torch.equal(ps[2 * n2s:].view(B, H // 2 + 1, -1)[:, :H // 2], pp[2 * n2:].view(B, H // 2, -1))) and \
        bool((ps[:2 * n2s].view(B, H // 2 + 1, -1)[:, H // 2] == 0xAB).all())
    ok = ok_compact and ok_rows and ok_pad and ok_pool
    print(json.dumps(dict(ok=ok, compact=ok_compact, rows=ok_rows, pad_zero=ok_pad, pooled_stack_out=ok_pool)))
    return 0 if ok else 1


def cmd_conv1(a):
    """conv1_1 (tensor-core im2col-in-smem kernel or the SIMT one) against float64 on the same uint8 image."""
    import torch
    from ctpn_b200 import _native as N
    dev = torch.device("cuda", 0)
    rs = np.random.RandomState(a.seed)
    im = rs.randint(0, 256, size=(a.B, a.H, a.W, 3)).astype(np.uint8)
    w = (rs.standard_normal((3, 3, 3, 64)) * (2.0 / 27) ** 0.5 / 75.0).astype(np.float32)
    b = (rs.standard_normal(64) * 0.1).astype(np.float32)
    means = np.array([102.9801, 115.9465, 122.7717])
    lut = (np.arange(256, dtype=np.float64)[:, None] - means[None, :]).astype(np.float32)
    imd, wd, bd, lutd = (torch.from_numpy(x).to(dev) for x in (im, w, b, lut))
    out = torch.zeros((a.planes, a.B, a.H, a.W, 64), dtype=torch.bfloat16, device=dev)
    fn = N.lib.ctpn_conv1_1 if a.impl == "simt" else N.lib.ctpn_conv1_1_tc
    N.check(fn(N.ptr(imd), 0, N.ptr(lutd), N.ptr(wd), N.ptr(bd), N.ptr(out), a.B, a.H, a.W, a.planes, N.stream_ptr()), "conv1_1")
    torch.cuda.synchronize()
    got = out.double().sum(0)
    x = torch.from_numpy(lut.astype(np.float64)[im.reshape(-1, 3), np.arange(3)].reshape(im.shape)).to(dev).permute(0, 3, 1, 2)
    wr = torch.from_numpy(w.astype(np.float64)).to(dev).permute(3, 2, 0, 1)
    y = torch.relu(torch.nn.functional.conv2d(x, wr, bd.double(), padding=1)).permute(0, 2, 3, 1)
    err = (got - y).abs().max().item()
    scale = y.abs().max().item()
    tol = {1: 1.2e-2, 2: 6e-5, 3: 3e-6}[a.planes] if a.impl != "simt" else {1: 4e-3, 2: 2e-5, 3: 2e-6}[a.planes]
    ok = bool(torch.isfinite(got).all().item()) and err <= tol * scale
    print(json.dumps(dict(ok=ok, max_err=err, scale=scale, rel=err / scale, tol=tol)))
    return 0 if ok else 1


def cmd_bilstm(a):
    import torch
    from ctpn_b200 import _native as N
    dev = torch.device("cuda", 0)
    rs = np.random.RandomState(a.seed)
    xproj = (rs.standard_normal((a.R, a.W, 1024)) * 1.0).astype(np.float32)
    wh = [(rs.uniform(-0.07, 0.07, (128, 512))).astype(np.float32) for _ in range(2)]
    xd = torch.from_numpy(xproj).to(dev)
    whd = [torch.from_numpy(w).to(dev) for w in wh]
    out = torch.zeros((a.planes, a.R, a.W, 256), dtype=torch.bfloat16, device=dev)
    N.check(N.lib.ctpn_bilstm_recurrent(N.ptr(xd), N.ptr(whd[0]), N.ptr(whd[1]), N.ptr(out), a.R, a.W, a.planes, N.stream_ptr()), "bilstm")
    torch.cuda.synchronize()
    got = out.double().sum(0).cpu().numpy()
    # float64 reference of the TF 1.3 LSTMCell recurrence (oracle.net_cpu.lstm_dir without the x-projection)
    ref = np.zeros((a.R, a.W, 256))
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))
    for d in range(2):
        h = np.zeros((a.R, 128)); c = np.zeros((a.R, 128))
        steps = range(a.W - 1, -1, -1) if d else range(a.W)
        for t in steps:
            gt = xproj[:, t, d * 512:(d + 1) * 512].astype(np.float64) + h @ wh[d].astype(np.float64)
            i, j, f, o = gt[:, :128], gt[:, 128:256], gt[:, 256:384], gt[:, 384:]
            c = sig(f + 1.0) * c + sig(i) * np.tanh(j)
            h = sig(o) * np.tanh(c)
            ref[:, t, d * 128:(d + 1) * 128] = h
    max_err = float(np.abs(got - ref).max())
    tol = {1: 4e-3, 2: 2e-5, 3: 5e-6}[a.planes]
    ok = bool(np.isfinite(got).all() and max_err <= tol)
    print(json.dumps(dict(ok=ok, max_err=max_err, tol=tol)))
    return 0 if ok else 1


def cmd_net_simt(a):
    """Whole network, tensor-core kernels vs the float32 SIMT reference kernels of the test library (same planes)."""
    import torch
    from ctpn_b200 import Engine
    from oracle import synth
    w = synth.make_weights(0)
    ims = np.stack([synth.make_image(20 + i, a.H, a.W) for i in range(a.B)])
    x = torch.from_numpy(ims).cuda()
    c1, b1 = Engine(w, planes=a.planes).forward_heads(x)
    c2, b2 = Engine(w, planes=a.planes, conv_simt=True).forward_heads(x)
    d = max(float((c1 - c2).abs().max()), float((b1 - b2).abs().max()))
    ok = d < a.tol
    print(json.dumps(dict(ok=bool(ok), head_diff=d, tol=a.tol)))
    return 0 if ok else 1


def cmd_proposals_generic(a):
    """CTPN_GENERIC_NMS=1 (test library): every image through the generic bitmask NMS; equals the oracle exactly."""
    import torch
    from ctpn_b200.engine import Engine
    from oracle import postproc, synth
    assert os.environ.get("CTPN_GENERIC_NMS") and os.environ.get("CTPN_B200_LIB") == "dbg"
    eng = Engine(None)
    H, W = 12, 18
    cls = np.concatenate([synth.make_head_outputs(200 + s, H, W)[0] for s in range(2)])
    box = np.concatenate([synth.make_head_outputs(200 + s, H, W)[1] for s in range(2)])
    info = np.array([[192, 100, 1.0], [192, 288, 1.0]], np.float32)
    rois, index, count = eng.proposals(torch.from_numpy(cls).cuda(), torch.from_numpy(box).cuda(), torch.from_numpy(info), cls_is_logit=False)
    ok = True
    for b in range(2):
        want, _, idx = postproc.proposal_layer(cls[b:b + 1], box[b:b + 1], info[b:b + 1], return_index=True)
        n = int(count[b])
        ok = ok and n == want.shape[0] and np.array_equal(index[b, :n].cpu().numpy(), idx) and np.array_equal(rois[b, :n].cpu().numpy(), want)
    print(json.dumps(dict(ok=bool(ok))))
    return 0 if ok else 1


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    c = sub.add_parser("conv")
    for k, d in dict(B=1, H=8, W=16, cin=64, cout=64, taps=9, planes=1, flags=0, seed=0, nonneg=0).items():
        c.add_argument("--" + k, type=int, default=d)
    c.add_argument("--impl", default="tc")
    c1 = sub.add_parser("conv1")
    for k, d in dict(B=1, H=37, W=45, planes=2, seed=0).items():
        c1.add_argument("--" + k, type=int, default=d)
    c1.add_argument("--impl", default="tc")
    l = sub.add_parser("bilstm")
    for k, d in dict(R=37, W=56, planes=2, seed=0).items():
        l.add_argument("--" + k, type=int, default=d)
    cq = sub.add_parser("conv_f16f8")
    for k, d in dict(B=1, H=8, W=16, cin=64, cout=64, taps=9, flags=0, seed=0).items():
        cq.add_argument("--" + k, type=int, default=d)
    cq.add_argument("--xscale", type=float, default=1.0)
    cs = sub.add_parser("conv_stack")
    for k, d in dict(B=3, H=37, W=56, cin=128, cout=128, seed=0).items():
        cs.add_argument("--" + k, type=int, default=d)
    ns = sub.add_parser("net_simt")
    for k, d in dict(B=3, H=128, W=192, planes=2).items():
        ns.add_argument("--" + k, type=int, default=d)
    ns.add_argument("--tol", type=float, default=5e-4)
    sub.add_parser("proposals_generic")
    a = ap.parse_args()
    return {"conv": cmd_conv, "conv_f16f8": cmd_conv_f16f8, "conv_stack": cmd_conv_stack, "conv1": cmd_conv1, "bilstm": cmd_bilstm, "net_simt": cmd_net_simt,
            "proposals_generic": cmd_proposals_generic}[a.cmd](a)


if __name__ == "__main__":
    sys.exit(main())
