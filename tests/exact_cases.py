"""Exact-arithmetic cases for the tensor-core convolutions (importable without a GPU): operands whose products and partial
sums are representable exactly in every accumulator the kernels use, and their float64 reference.

With such operands the correct output of conv_tc_kernel / conv1_tc_kernel is ONE float32 number per element, whatever the
order of the tensor core's adds, so the kernel must reproduce it bit for bit; a dropped, doubled or misplaced tap, channel
slice, plane pair or cross MMA changes an output instead of hiding below a tolerance.

bf16 planes (ctpn_conv3x3, P planes): every plane of x and w holds small integers, drawn independently per plane (the kernel
does not care that planes are residuals, and independent planes make each pair (i, j) distinguishable).  Every 8th output
channel has a bias of 2^18 + an odd integer, so its outputs carry 19 significant bits and the bf16 split of the output
needs all three planes (the outputs of small integers alone would leave the third plane zero).  The reference is
    y = sum_{i + j < P} conv(x_i, w_j) + bias  -> ReLU -> 2x2 max-pool
(the SIMT reference kernel multiplies the plane sums, i.e. every pair: pairs="all").
F16F8 (ctpn_conv3x3_f16f8): raw operand bytes.  The fp16 plane holds integers, the e4m3 value and residual halves small
e4m3-exact integers, sparse enough for the cross bound; activation rows are value | residual, weight rows residual | value
(include/ctpn_b200.h).  y = conv(h_a, h_w) * inv_main + (conv(v_a, r_w) + conv(r_a, v_w)) * inv_cross + bias with
inv_cross != inv_main, so a mix-up of the main and cross accumulators shows.
conv1_1 (ctpn_conv1_1_tc, K = 27 + a bias row): LUT / blob values and weights with 9-10 significant bits, so both cross
pairs of P = 2 are non-zero.  P = 3 would need 17-bit significands, which break the 2^20 bound below; it is left to the
float64 bound of tests/gpu_checks.py (3e-6 of max |y|, which resolves the third plane: 2^-16).

Preconditions (check_preconditions, asserted before any launch), in units of the operands' common quantum:
  * bf16 / fp16 accumulators: sum |products| <= 2^20 per output (float32 holds 2^24);
  * e4m3 cross accumulator: sum |products| <= 2^12 per output (the e4m3 wgmma is publicly reported to keep ~14 significant
    bits when it adds into float32).  The operands aim at a mean of CROSS_FILL (a quarter) of that bound; two cases of
    tests/test_exact_gpu.py raise it until the largest per-output cross sums come within 5 % of the bound.  On an H100
    (700 W limit) both are exact with sums of up to 4004 and 3952 units, so the bound holds as measured;
  * main * inv_main, cross * inv_cross, their sum and the biased value are each exactly float32 (the __fmaf_rn /
    bias add of the conv_tc epilogue);
  * every plane of each bf16 plane output the checks compare (P planes, or the two of CTPN_F_OUT_BF16X2) is non-zero in
    every output tile, so a plane stored as zeros, or a split stopped early, fails the comparison in any tile.
Coverage (coverage): for every structural term -- each plane pair (or main / cross product), each tap, each 64-channel
block, each K = 16 slice (bf16 / fp16; all pairs of the slice together) or K = 32 slice of each e4m3 cross product, and
the bias -- removing it from the reference changes at least one output of every output tile (16 x 8 input pixels, or 128
for taps = 1, x 64 channels: every BN tile contains whole 64-channel groups).  Row-stacked layouts are checked on the
plain layout's tiles."""
import math

import numpy as np
import torch

F_RELU, F_POOL, F_F32, F_OUT_BF16X2, F_STACK_IN, F_STACK_OUT, F_PROMOTE = 1, 2, 4, 8, 16, 32, 64
ACC_BOUND = 2 ** 20
CROSS_BOUND = 2 ** 12
CROSS_FILL = 0.25                                # default mean cross sum, as a fraction of CROSS_BOUND
INV_MAIN, INV_CROSS = 2.0 ** -5, 2.0 ** -2      # F16F8 epilogue scales: distinct powers of two
MAX_CHUNK = 1 << 25                              # float64 elements per batch of slice contributions


# ---- cases -------------------------------------------------------------------------------------------------------------

def conv(B, H, W, cin, cout, taps, planes, flags):
    return dict(kind="conv", B=B, H=H, W=W, cin=cin, cout=cout, taps=taps, planes=planes, flags=flags)


def f16f8(B, H, W, cin, cout, taps, flags, cross_fill=None):
    """cross_fill: mean per-output cross sum as a fraction of CROSS_BOUND (default CROSS_FILL)."""
    c = dict(kind="conv_f16f8", B=B, H=H, W=W, cin=cin, cout=cout, taps=taps, planes=2, flags=flags)
    if cross_fill is not None:
        c["cross_fill"] = cross_fill
    return c


def argv(case):
    """Command line of tests/exact_checks.py for a case."""
    keys = ["B", "H", "W", "cin", "cout", "taps"] + (["planes"] if case["kind"] == "conv" else []) + ["flags"]
    out = [case["kind"]]
    for k in keys:
        out += ["--" + k, case[k]]
    if "cross_fill" in case:
        out += ["--cross_fill", case["cross_fill"]]
    return out


RELU, POOL, F32, PROMOTE = F_RELU, F_POOL, F_F32, F_PROMOTE
# One exact case per conv_tc instantiation, keyed like tests/test_kernel_variants_gpu.VARIANTS
# (taps, f16f8, planes, BN, mc, promote), at the same shapes and flags.
VARIANT_CASES = {
    (9, 1, 2, 128, 1, 0): f16f8(1, 75, 112, 256, 512, 9, RELU),
    (9, 1, 2, 64, 1, 0): f16f8(2, 50, 70, 64, 64, 9, RELU | POOL),
    (9, 1, 2, 128, 0, 0): f16f8(1, 9, 6, 512, 512, 9, RELU),
    (9, 1, 2, 64, 0, 0): f16f8(1, 16, 8, 64, 64, 9, RELU | POOL),
    (1, 1, 2, 128, 0, 0): f16f8(1, 1, 300, 256, 128, 1, 0),
    (1, 1, 2, 64, 0, 0): f16f8(1, 1, 2072, 512, 64, 1, 0),
    (9, 0, 3, 128, 1, 1): conv(1, 75, 112, 128, 256, 9, 3, RELU | PROMOTE),
    (9, 0, 3, 64, 1, 1): conv(1, 300, 450, 64, 64, 9, 3, RELU | POOL | PROMOTE),
    (9, 0, 3, 64, 0, 1): conv(1, 16, 8, 512, 512, 9, 3, RELU | PROMOTE),
    (1, 0, 3, 128, 0, 1): conv(1, 1, 2072, 256, 512, 1, 3, PROMOTE),
    (1, 0, 3, 64, 0, 1): conv(1, 1, 2072, 512, 64, 1, 3, F32 | PROMOTE),
    (9, 0, 1, 256, 1, 0): conv(2, 19, 21, 256, 512, 9, 1, RELU | POOL),
    (9, 0, 1, 128, 1, 0): conv(1, 150, 225, 128, 128, 9, 1, RELU | POOL),
    (9, 0, 1, 64, 1, 0): conv(1, 300, 450, 64, 64, 9, 1, RELU | POOL),
    (9, 0, 2, 128, 1, 0): conv(1, 37, 56, 512, 512, 9, 2, RELU),
    (9, 0, 2, 64, 1, 0): conv(2, 50, 70, 64, 64, 9, 2, RELU | POOL),
    (9, 0, 3, 128, 1, 0): conv(1, 75, 112, 256, 512, 9, 3, RELU),
    (9, 0, 3, 64, 1, 0): conv(3, 75, 112, 64, 64, 9, 3, RELU | POOL),
    (9, 0, 1, 256, 0, 0): conv(1, 13, 7, 256, 256, 9, 1, RELU | POOL),
    (9, 0, 1, 128, 0, 0): conv(1, 8, 8, 128, 128, 9, 1, RELU | POOL),
    (9, 0, 1, 64, 0, 0): conv(1, 11, 5, 64, 64, 9, 1, RELU | F32),
    (9, 0, 2, 128, 0, 0): conv(1, 9, 6, 512, 512, 9, 2, RELU | POOL),
    (9, 0, 2, 64, 0, 0): conv(1, 16, 8, 64, 64, 9, 2, RELU),
    (9, 0, 3, 128, 0, 0): conv(1, 12, 8, 256, 256, 9, 3, RELU | POOL),
    (9, 0, 3, 64, 0, 0): conv(1, 16, 8, 64, 64, 9, 3, RELU | POOL),
    (1, 0, 1, 256, 0, 0): conv(1, 1, 2072, 512, 1024, 1, 1, F32),
    (1, 0, 1, 128, 0, 0): conv(1, 1, 333, 256, 128, 1, 1, 0),
    (1, 0, 1, 64, 0, 0): conv(1, 1, 2072, 512, 64, 1, 1, F32),
    (1, 0, 2, 128, 0, 0): conv(1, 1, 2072, 256, 512, 1, 2, 0),
    (1, 0, 2, 64, 0, 0): conv(1, 1, 777, 512, 64, 1, 2, F32),
    (1, 0, 3, 128, 0, 0): conv(1, 1, 2072, 512, 1024, 1, 3, F32),
    (1, 0, 3, 64, 0, 0): conv(1, 1, 2072, 512, 64, 1, 3, F32),
}


def macs(case):
    return case["B"] * case["H"] * case["W"] * case["taps"] * case["cin"] * case["cout"]


# ---- operands ----------------------------------------------------------------------------------------------------------

def _ints(g, shape, lo, hi):
    return torch.randint(lo, hi + 1, shape, generator=g).double()


def _sparse_e4m3_ints(g, shape, density):
    """Integers in {0, +-1, +-2} (e4m3-exact), non-zero with the given probability."""
    mag = torch.randint(1, 3, shape, generator=g).double()
    sign = torch.randint(0, 2, shape, generator=g).double() * 2 - 1
    return mag * sign * (torch.rand(shape, generator=g, dtype=torch.float64) < density).double()


def _bias(g, n, wide=False):
    """Non-zero small integers of both signs.  wide: every 8th channel (c % 8 == 3) gets 2^18 + an odd integer below 2^12
    instead, so its outputs have 19 significant bits: a bf16 plane split of them needs all three planes (p2 holds bits
    below the 16th), while every output stays an exact float32 integer."""
    b = _ints(g, (n,), 1, 8)
    b = b * (torch.randint(0, 2, (n,), generator=g).double() * 2 - 1)
    if wide:
        b[3::8] = 2.0 ** 18 + (2 * torch.randint(0, 2 ** 11, (len(range(3, n, 8)),), generator=g) + 1).double()
    return b


def bf16_operands(case, seed=0):
    """x [P][B][H][W][Cin], w [P][taps][Cin][Cout] (TF layout per plane): float64 integers in [-3, 3]; bias [Cout]: _bias
    with the wide channels."""
    g = torch.Generator().manual_seed(seed)
    P = case["planes"]
    x = _ints(g, (P, case["B"], case["H"], case["W"], case["cin"]), -3, 3)
    w = _ints(g, (P, case["taps"], case["cin"], case["cout"]), -3, 3)
    return dict(x=x, w=w, bias=_bias(g, case["cout"], wide=True))


def f16f8_operands(case, seed=0):
    """fp16 plane integers in [-7, 7]; e4m3 halves sparse integers, the density set so that the mean cross sum is
    case["cross_fill"] (default CROSS_FILL) of CROSS_BOUND.  Activations [B][H][W][Cin], weights [taps][Cin][Cout]."""
    g = torch.Generator().manual_seed(seed)
    B, H, W, C, Co, T = case["B"], case["H"], case["W"], case["cin"], case["cout"], case["taps"]
    pairs = 2 * T * C                                  # cross products per output
    fill = case.get("cross_fill", CROSS_FILL)
    density = min(0.5, math.sqrt(CROSS_BOUND * fill / (pairs * 2.25)))   # E|v r| = density^2 * 1.5^2
    return dict(h_a=_ints(g, (B, H, W, C), -7, 7), v_a=_sparse_e4m3_ints(g, (B, H, W, C), density),
                r_a=_sparse_e4m3_ints(g, (B, H, W, C), density),
                h_w=_ints(g, (T, C, Co), -7, 7), v_w=_sparse_e4m3_ints(g, (T, C, Co), density),
                r_w=_sparse_e4m3_ints(g, (T, C, Co), density), bias=_bias(g, Co), inv_main=INV_MAIN, inv_cross=INV_CROSS)


def products(case, ops, pairs="tc"):
    """The reference as a list of groups [(name, [(x [B,H,W,Cin], w [taps,Cin,Cout], scale)], slice width)]: each group is
    one accumulator's structural slice family (coverage removes whole groups, their K slices, taps and blocks)."""
    if case["kind"] == "conv_f16f8":
        return [("main", [(ops["h_a"], ops["h_w"], ops["inv_main"])], 16),
                ("value_x_residual", [(ops["v_a"], ops["r_w"], ops["inv_cross"])], 32),
                ("residual_x_value", [(ops["r_a"], ops["v_w"], ops["inv_cross"])], 32)]
    P = ops["x"].shape[0]
    pl = [(i, j) for i in range(P) for j in range(P) if pairs == "all" or i + j < P]
    return [("pairs", [(ops["x"][i], ops["w"][j], 1.0) for i, j in pl], 16)]


def plane_pairs(case, ops, pairs="tc"):
    """Per-pair terms (removed one at a time by the coverage check): [(name, [(x, w, scale)])]."""
    if case["kind"] == "conv_f16f8":
        return [(name, prods) for name, prods, _ in products(case, ops)]
    P = ops["x"].shape[0]
    return [("x%d_w%d" % (i, j), [(ops["x"][i], ops["w"][j], 1.0)]) for i in range(P) for j in range(P)
            if pairs == "all" or i + j < P]


# ---- float64 convolution by taps and channel slices ---------------------------------------------------------------------

def _shifted(x, tap, taps):
    """x [B,H,W,C] -> the input seen by filter tap `tap` at every output pixel (SAME zero padding)."""
    if taps == 1:
        return x
    ky, kx = divmod(tap, 3)
    xp = torch.nn.functional.pad(x, (0, 0, 1, 1, 1, 1))
    return xp[:, ky:ky + x.shape[1], kx:kx + x.shape[2], :]


def partial(prods, taps, tap=None, c0=0, c1=None, absolute=False):
    """sum over prods of scale * x . w restricted to one tap (or all) and channels [c0, c1): [B,H,W,Cout] float64."""
    out = None
    for x, w, s in prods:
        cc = x.shape[-1] if c1 is None else c1
        for t in (range(taps) if tap is None else [tap]):
            xs, ws = _shifted(x, t, taps)[..., c0:cc], w[t, c0:cc]
            if absolute:
                xs, ws = xs.abs(), ws.abs()
            v = torch.matmul(xs, ws) * s
            out = v if out is None else out + v
    return out


def slice_contributions(prods, taps, width):
    """Yields (tap, c0, contributions [n, B,H,W,Cout]) for every K slice of `width` channels, in batches."""
    x0 = prods[0][0]
    B, H, W, C = x0.shape
    Co = prods[0][1].shape[-1]
    ns = C // width
    per = max(1, min(ns, MAX_CHUNK // max(1, B * H * W * Co)))
    for t in range(taps):
        for s0 in range(0, ns, per):
            s1 = min(ns, s0 + per)
            acc = None
            for x, w, sc in prods:
                xs = _shifted(x, t, taps)[..., s0 * width:s1 * width].reshape(B, H, W, s1 - s0, width)
                ws = w[t, s0 * width:s1 * width].reshape(s1 - s0, width, Co)
                v = torch.einsum("bhwsk,skn->sbhwn", xs, ws) * sc
                acc = v if acc is None else acc + v
            yield t, s0 * width, acc


def post(case, y):
    """+ReLU, 2x2/2 max-pool of a pre-activation [..., B, H, W, C] (leading dims allowed)."""
    f = case["flags"]
    if f & F_RELU:
        y = y.clamp_min(0.0)
    if f & F_POOL:
        lead, (B, H, W, C) = y.shape[:-4], y.shape[-4:]
        Ho, Wo = H // 2, W // 2
        y = y[..., :2 * Ho, :2 * Wo, :].reshape(*lead, B, Ho, 2, Wo, 2, C).amax(dim=(-4, -2))
    return y


def preact(case, ops, pairs="tc"):
    """Pre-activation reference: sum of every group + bias, [B,H,W,Cout] float64."""
    y = None
    for _, prods, _ in products(case, ops, pairs):
        v = partial(prods, case["taps"])
        y = v if y is None else y + v
    return y + ops["bias"]


def reference(case, ops, pairs="tc"):
    return post(case, preact(case, ops, pairs))


# ---- preconditions -----------------------------------------------------------------------------------------------------

def _exact_f32(t):
    return bool(torch.equal(t.float().double(), t))


def check_preconditions(case, ops, pairs="tc"):
    """dict of the measured bounds and a list of violated preconditions (empty = exact)."""
    taps, bad, res = case["taps"], [], {}
    groups = products(case, ops, pairs)
    if case["kind"] == "conv_f16f8":
        main = partial(groups[0][1], taps) / ops["inv_main"]
        cross = (partial(groups[1][1], taps) + partial(groups[2][1], taps)) / ops["inv_cross"]
        amain = partial(groups[0][1], taps, absolute=True) / ops["inv_main"]
        across = (partial(groups[1][1], taps, absolute=True) + partial(groups[2][1], taps, absolute=True)) / ops["inv_cross"]
        res.update(acc_units=amain.max().item(), cross_units=across.max().item())
        if res["acc_units"] > ACC_BOUND:
            bad.append("fp16 main accumulator %g > 2^20 units" % res["acc_units"])
        if res["cross_units"] > CROSS_BOUND:
            bad.append("e4m3 cross accumulator %g > 2^12 units" % res["cross_units"])
        for name, t in (("main", main), ("cross", cross)):
            if not torch.equal(t, t.round()):
                bad.append("%s accumulator not integral" % name)
        m, c = main * ops["inv_main"], cross * ops["inv_cross"]
        for name, t in (("main*inv_main", m), ("cross*inv_cross", c), ("sum", m + c), ("biased", m + c + ops["bias"])):
            if not _exact_f32(t):
                bad.append("%s not exact in float32" % name)
    else:
        a = None
        for x, w, s in groups[0][1]:
            v = partial([(x, w, s)], taps, absolute=True)
            a = v if a is None else a + v
        res["acc_units"] = a.max().item()
        if res["acc_units"] > ACC_BOUND:
            bad.append("bf16 accumulator %g > 2^20 units" % res["acc_units"])
        for name, t in (("accumulator", preact(case, ops, pairs) - ops["bias"]), ("biased", preact(case, ops, pairs))):
            if not (torch.equal(t, t.round()) and _exact_f32(t)):
                bad.append("%s not an exact float32 integer" % name)
    if case["flags"] & F_RELU:
        y = preact(case, ops, pairs)
        res["relu_clipped"] = float((y < 0).double().mean().item())
        if not res["relu_clipped"] > 0:
            bad.append("ReLU clips nothing")
    # the bf16 plane outputs the checks compare: P planes (bf16), the CTPN_F_OUT_BF16X2 pair (F16F8)
    _check_planes(case, reference(case, ops, pairs), 2 if case["kind"] == "conv_f16f8" else case["planes"], res, bad)
    return res, bad


def _check_planes(case, y, planes, res, bad):
    """Every plane of the bf16 split of the outputs y is non-zero somewhere in every output tile, so an output plane that a
    kernel stored as zeros (or a split stopped early) fails the bit-for-bit comparison in any tile."""
    split = split_planes(y.float(), planes).double()
    res["zero_plane_tiles"] = [int((~tiles_changed(case, torch.zeros_like(pl), pl)).sum().item()) for pl in split]
    for k, n in enumerate(res["zero_plane_tiles"]):
        if n:
            bad.append("output plane %d is zero in %d tiles" % (k, n))


# ---- coverage ----------------------------------------------------------------------------------------------------------

def tile_geometry(case):
    """(rows, cols) of one pixel tile in OUTPUT coordinates."""
    s = 2 if case["flags"] & F_POOL else 1
    return (16 // s, 8 // s) if case["taps"] == 9 else (1, 128)


def tiles_changed(case, ref_out, new_out):
    """[..., B, Ho, Wo, C] outputs -> bool [..., B, tiles_y, tiles_x, C / 64]: some output of the tile differs."""
    th, tw = tile_geometry(case)
    d = new_out != ref_out
    lead, (B, Ho, Wo, C) = d.shape[:-4], d.shape[-4:]
    ty, tx = -(-Ho // th), -(-Wo // tw)
    d = torch.nn.functional.pad(d.to(torch.uint8), (0, 0, 0, tx * tw - Wo, 0, ty * th - Ho))
    return d.reshape(*lead, B, ty, th, tx, tw, C // 64, 64).amax(dim=(-5, -3, -1)).bool()


def coverage(case, ops, pairs="tc"):
    """{term family: number of (term, output tile) pairs where removing the term changes nothing} and the tile count."""
    taps, C = case["taps"], case["cin"]
    y = preact(case, ops, pairs)
    ref = post(case, y)
    miss = {}

    def count(name, contrib):       # contrib [n, B,H,W,Co] or [B,H,W,Co]
        ch = tiles_changed(case, ref, post(case, y - contrib))
        miss[name] = miss.get(name, 0) + int((~ch).sum().item())
        return ch

    groups = products(case, ops, pairs)
    allprods = [p for _, prods, _ in groups for p in prods]
    ntiles = tiles_changed(case, ref, ref).numel()
    for name, prods in plane_pairs(case, ops, pairs):
        count("pair " + name, partial(prods, taps))
    for t in range(taps):
        count("tap", partial(allprods, taps, tap=t))
    for c0 in range(0, C, 64):
        count("block", partial(allprods, taps, c0=c0, c1=c0 + 64))
    for name, prods, width in groups:
        for _, _, contrib in slice_contributions(prods, taps, width):
            count("k%d slice %s" % (width, name), contrib)
    count("bias", ops["bias"].expand_as(y))
    return miss, ntiles


# ---- device encodings --------------------------------------------------------------------------------------------------

def bf16_inputs(ops):
    """(activation planes [P][B][H][W][Cin] bf16, weight planes [P][Cout][taps][Cin] bf16): exact conversions."""
    return ops["x"].to(torch.bfloat16).contiguous(), ops["w"].permute(0, 3, 1, 2).to(torch.bfloat16).contiguous()


def stacked(x):
    """[P][B][H][W][C] -> [P][B][H + 1][W][C] with one zero row after every image (CTPN_F_STACK_IN)."""
    P, B, H, W, C = x.shape
    out = torch.zeros((P, B, H + 1, W, C), dtype=x.dtype, device=x.device)
    out[:, :, :H] = x
    return out


def _e4m3_bytes(v):
    return v.float().to(torch.float8_e4m3fn).view(torch.uint8)


def f16f8_inputs(ops):
    """(activation bytes, weight bytes) in the F16F8 plane layouts: [fp16 plane | e4m3 plane]."""
    ha, va, ra = ops["h_a"], ops["v_a"], ops["r_a"]
    lead, C = ha.shape[:-1], ha.shape[-1]
    act_cross = torch.cat([_e4m3_bytes(va).reshape(lead + (C // 64, 64)), _e4m3_bytes(ra).reshape(lead + (C // 64, 64))], -1)
    act = torch.cat([ha.to(torch.float16).contiguous().view(torch.uint8).reshape(-1), act_cross.reshape(-1)])
    hw, vw, rw = (ops[k].permute(2, 0, 1).contiguous() for k in ("h_w", "v_w", "r_w"))    # [Cout][taps][Cin]
    lead, C = hw.shape[:-1], hw.shape[-1]
    w_cross = torch.cat([_e4m3_bytes(rw).reshape(lead + (C // 64, 64)), _e4m3_bytes(vw).reshape(lead + (C // 64, 64))], -1)
    wt = torch.cat([hw.to(torch.float16).contiguous().view(torch.uint8).reshape(-1), w_cross.reshape(-1)])
    return act, wt


def split_planes(y32, planes):
    """float32 tensor -> [P, ...] bf16 planes (the kernels' rule: p_k = bf16_rn(remainder), remainder -= p_k)."""
    out, r = [], y32.clone()
    for _ in range(planes):
        h = r.to(torch.bfloat16)
        out.append(h)
        r = r - h.to(torch.float32)
    return torch.stack(out, 0)


# ---- conv1_1 -----------------------------------------------------------------------------------------------------------

def conv1_operands(B, H, W, seed=0, blob=False):
    """conv1_1 inputs: a uint8 image and LUT [256][3] (or a float32 blob [B][H][W][3]), weights [3][3][3][64], bias [64].
    Channel 0 of the input and channels 1, 2 of the weights hold integers in [-15, 15]; channels 1, 2 of the input and
    channel 0 of the weights hold, half of the time, odd 9-10-bit integers (257..1023), whose bf16 residual plane is not
    zero.  Wide values never meet in one product, which keeps every output within ACC_BOUND."""
    g = torch.Generator().manual_seed(seed)

    def wide_or_small(shape):
        small = _ints(g, shape, -15, 15)
        wide = (2 * torch.randint(128, 512, shape, generator=g) + 1).double()
        wide = wide * (torch.randint(0, 2, shape, generator=g).double() * 2 - 1)
        return torch.where(torch.rand(shape, generator=g) < 0.5, wide, small)
    w = _ints(g, (3, 3, 3, 64), -15, 15)
    w[:, :, 0] = wide_or_small((3, 3, 64))
    bias = _bias(g, 64)
    if blob:
        x = _ints(g, (B, H, W, 3), -15, 15)
        x[..., 1:] = wide_or_small((B, H, W, 2))
        return dict(x=x, w=w, bias=bias)
    lut = _ints(g, (256, 3), -15, 15)
    lut[:, 1:] = wide_or_small((256, 2))
    im = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    x = lut[im.long(), torch.arange(3)]
    return dict(x=x, w=w, bias=bias, lut=lut, im=im)


def conv1_terms(ops, planes):
    """conv1_1 as the kernel computes it: K = 27 inputs (k = (ky * 3 + kx) * 3 + c) plus the bias row (A = 1), both sides
    split into bf16 planes, pairs i + j < P.  Returns (A [P][B][H][W][28], Wk [P][28][64]) float64."""
    x, w, bias = ops["x"], ops["w"], ops["bias"]
    B, H, W, _ = x.shape
    xp = torch.nn.functional.pad(x, (0, 0, 1, 1, 1, 1))
    cols = [xp[:, ky:ky + H, kx:kx + W, c] for ky in range(3) for kx in range(3) for c in range(3)]
    A = torch.stack(cols + [torch.ones_like(cols[0])], -1)
    Wk = torch.cat([w.reshape(27, 64), bias.view(1, 64)], 0)
    Ap = split_planes(A.float(), planes).double()
    Wp = split_planes(Wk.float(), planes).double()
    return Ap, Wp


def conv1_case(planes):
    return dict(kind="conv1", taps=9, flags=F_RELU, planes=planes)


def conv1_preact(Ap, Wp, drop=None):
    """sum_{i + j < P} A_i . W_j, optionally without some terms: drop(i, j) -> a [28] mask of the k to leave out."""
    P = Ap.shape[0]
    y = 0
    for i in range(P):
        for j in range(P - i):
            Wj = Wp[j]
            if drop is not None:
                Wj = Wj * (1.0 - drop(i, j)).view(-1, 1)
            y = y + torch.matmul(Ap[i], Wj)
    return y


def conv1_check(ops, planes):
    """(bounds, violated preconditions, uncovered (term, tile) counts, tile count) for ctpn_conv1_1_tc."""
    Ap, Wp = conv1_terms(ops, planes)
    P = planes
    res, bad = {}, []
    for name, t in (("inputs", Ap), ("weights", Wp)):
        if not torch.equal(t, t.round()):
            bad.append("%s not integral" % name)
    a = sum(torch.matmul(Ap[i].abs(), Wp[j].abs()) for i in range(P) for j in range(P - i))
    res["acc_units"] = a.max().item()
    if res["acc_units"] > ACC_BOUND:
        bad.append("accumulator %g > 2^20 units" % res["acc_units"])
    y = conv1_preact(Ap, Wp)
    res["relu_clipped"] = float((y < 0).double().mean().item())
    if not res["relu_clipped"] > 0:
        bad.append("ReLU clips nothing")
    case = conv1_case(P)
    ref = post(case, y)
    _check_planes(case, ref, P, res, bad)
    miss = {}
    ones = torch.ones(28, dtype=torch.float64, device=y.device)
    zero = torch.zeros(28, dtype=torch.float64, device=y.device)

    def count(name, drop):
        ch = tiles_changed(case, ref, post(case, conv1_preact(Ap, Wp, drop)))
        miss[name] = miss.get(name, 0) + int((~ch).sum().item())
    for pi in range(P):
        for pj in range(P - pi):
            count("pair x%d_w%d" % (pi, pj), lambda i, j, pi=pi, pj=pj: ones if (i, j) == (pi, pj) else zero)
    for t in range(9):
        m = zero.clone()
        m[3 * t:3 * t + 3] = 1
        count("tap", lambda i, j, m=m: m)
    for k0 in (0, 16):
        m = zero.clone()
        m[k0:k0 + 16] = 1
        count("k16 slice", lambda i, j, m=m: m)
    m = zero.clone()
    m[27] = 1
    count("bias", lambda i, j, m=m: m)
    return res, bad, miss, tiles_changed(case, ref, ref).numel(), y
