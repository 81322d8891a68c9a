"""Case builders for the proposal-layer and NMS path tests (tests/test_proposal_cases_cpu.py checks them without a GPU,
tests/test_proposal_paths_gpu.py and tests/proposal_checks.py run them on the device), and a restatement of the rule by
which ctpn_proposals picks its NMS path.

Everything here is plain numpy on the CPU oracle's float32 arithmetic (oracle/postproc.py); exact classifications use
fractions.Fraction on the float32 values the kernels see.
"""
from fractions import Fraction

import numpy as np

from oracle import postproc

F32 = np.float32

# ---- dispatch rule: csrc/proposal.cu, column_smem_bytes() and proposals_run() -----------------------------------------
STATIC_SMEM = 48 * 1024    # proposals_run: col_smem > 48 KB needs the opt-in attribute
OPTIN_SMEM = 200 * 1024    # proposals_run: try_columns needs col_smem <= 200 KB (and H * 10 <= 2048)
BUCKET_MAX_W = 256         # proposals_run: bucket = try_columns && W <= 256 (col_start has 257 entries per image)


def column_smem_bytes(H):
    """csrc/proposal.cu column_smem_bytes(): one column's boxes, pairwise mask, areas and positions."""
    cap = H * 10
    wc = (cap + 63) // 64
    return cap * 16 + cap * wc * 8 + cap * 4 + cap * 4


def dispatch(H, W, feat_stride=16, lib=None):
    """(nms, sort) that proposals_run takes for an H x W map.  nms: 'column-static' | 'column-optin' | 'generic-all';
    sort: 'bucketed' (the sort kernel's extra column pass) | 'gathered' (each column CTA gathers from the score order) |
    None (no column NMS).  lib: None for the product library, else the environment of the test library, whose
    CTPN_GENERIC_NMS / CTPN_COLUMN_GATHER switches force the generic NMS / the gather."""
    env = lib or {}
    smem = column_smem_bytes(H)
    columns = (feat_stride >= 16 and smem <= OPTIN_SMEM and H * 10 <= 2048 and W <= 65535
               and not env.get("CTPN_GENERIC_NMS"))
    if not columns:
        return "generic-all", None
    nms = "column-static" if smem <= STATIC_SMEM else "column-optin"
    return nms, ("bucketed" if W <= BUCKET_MAX_W and not env.get("CTPN_COLUMN_GATHER") else "gathered")


def decoded(cls, bbox, info, feat_stride=16, py2=False, min_size=8, exp_mode="rounded"):
    """Decode + clip + size filter of one image exactly as postproc.proposal_layer does: (boxes [NA,4], scores [NA],
    valid [NA] bool), rows in anchor (h, w, a) order."""
    H, W = cls.shape[1:3]
    info = np.asarray(info, F32).reshape(-1, 3)[0]
    props = postproc.decode_boxes(postproc.shifted_anchors(H, W, feat_stride, py2), np.asarray(bbox, F32).reshape(-1, 4),
                                  exp_mode)
    props = postproc.clip(props, info[0], info[1])
    valid = np.zeros(len(props), bool)
    valid[postproc.size_filter(props, F32(min_size) * info[2])] = True
    return props, np.asarray(cls, F32).reshape(-1, 10, 2)[:, :, 1].reshape(-1), valid


def sorted_candidates(cls, bbox, info, pre=0, **kw):
    """What the proposal layer returns when NMS suppresses nothing (threshold 1.0, no post cut): (boxes, scores, index)
    of the valid boxes in postproc.order_desc order, cut at pre when pre > 0."""
    boxes, scores, valid = decoded(cls, bbox, info, **kw)
    idx = np.nonzero(valid)[0]
    order = idx[postproc.order_desc(scores[idx])]
    if pre > 0:
        order = order[:pre]
    return boxes[order], scores[order], order


def gate_triggers(cls, bbox, info, nms_thresh=0.7, feat_stride=16, py2=False, min_size=8):
    """The decode kernel's per-image structure check (csrc/proposal.cu proposal_decode_kernel): the set of triggers that
    some valid box trips -- 'x1' (x1 != anchor x1), 'x2' (x2 > anchor x1 + stride), 'width' ((2 ws - 1) * thresh <= 1).
    A non-empty set sends the image to the generic NMS."""
    H, W = cls.shape[1:3]
    boxes, _, valid = decoded(cls, bbox, info, feat_stride, py2, min_size)
    ax1 = postproc.shifted_anchors(H, W, feat_stride, py2)[:, 0].astype(F32)
    b = boxes[valid]
    ax1 = ax1[valid]
    ws = b[:, 2] - b[:, 0] + F32(1)
    out = set()
    if (b[:, 0] != ax1).any():
        out.add("x1")
    if (b[:, 2] > ax1 + F32(feat_stride)).any():
        out.add("x2")
    if ((F32(2) * ws - F32(1)) * F32(nms_thresh) <= F32(1)).any():
        out.add("width")
    return out


# ---- head builders ---------------------------------------------------------------------------------------------------
def random_heads(seed, B, H, W, quantise=None):
    """[B,H,W,20] fg/bg probabilities and [B,H,W,40] deltas from oracle.synth (pairwise-distinct scores unless quantised
    to multiples of 1 / quantise)."""
    from oracle import synth
    cls, box = [], []
    for b in range(B):
        c, d = synth.make_head_outputs(seed + b, H, W, unique=quantise is None)
        if quantise:
            c = (np.round(c * quantise) / quantise).astype(F32)
        cls.append(c[0])
        box.append(d[0])
    return np.stack(cls), np.stack(box)


def exact_heads(H, W, B=1):
    """All-zero deltas (dy = dh = 0: every box is its anchor, decoded exactly) and all-zero scores, to be filled in."""
    return np.zeros((B, H, W, 20), F32), np.zeros((B, H, W, 40), F32)


def ulp_pairs(base, count, parity):
    """count score pairs (lo, hi) with hi = nextafter(lo, +inf) and lo's last mantissa bit == parity."""
    out = []
    u = np.array([base], F32).view(np.uint32)[0]
    u = u - (u & 1) + parity
    for k in range(count):
        lo = np.array([u + 4 * k], np.uint32).view(F32)[0]
        out.append((lo, np.nextafter(lo, F32(np.inf))))
    return out


def ulp_pair_heads(H, W, per_parity=40, seed=0):
    """Probabilities quantised to 1/64 plus score pairs one float32 ulp apart, the higher one at the larger anchor index,
    in both parities of the last mantissa bit.  A sort key that drops the lowest bit orders such a pair by index, i.e.
    the wrong way round.  Returns (cls, bbox, pair_index [n,2] of (lower-score index, higher-score index))."""
    rs = np.random.RandomState(seed)
    cls, bbox = exact_heads(H, W)
    bbox[..., 1::4] = (rs.randint(-8, 9, bbox[..., 1::4].shape) / 16.0).astype(F32)   # dy: shifts, still exact
    fg = (rs.randint(1, 64, (H * W * 10,)) / 64.0).astype(F32)
    pairs = ulp_pairs(F32(0.3), per_parity, 0) + ulp_pairs(F32(0.55), per_parity, 1)
    slots = rs.choice(H * W * 10 // 2, len(pairs), replace=False) * 2        # anchor indices 2k, 2k+1
    for s, (lo, hi) in zip(slots, pairs):
        fg[s], fg[s + 1] = lo, hi
    cls[0, ..., 1::2] = fg.reshape(H, W, 10)
    cls[0, ..., 0::2] = F32(1) - cls[0, ..., 1::2]
    return cls, bbox, np.stack([slots, slots + 1], 1)


# ---- borderline IoU pairs --------------------------------------------------------------------------------------------
BAND = Fraction(1, 2 ** 20)      # csrc/nms_iou.cuh iou_above: |inter - t * u| <= 2^-20 max(inter, u) -> IEEE division


def required_classes(thresh, integer_boxes=False):
    """The borderline classes (see classify) a pair set must cover at float32(thresh).  Near 0.5 no float32 quotient
    other than an exact 0.5 rounds to 0.5 (the neighbours of an inter / u of float32 terms lie 2^-25 or more away), so
    there 'exact' takes the place of 'eq_above'.  For integer boxes (the generic pairs) 'eq_above' at float32(0.2) would
    need a union of 2^24 or more: 0 < ov / u - float32(0.2) <= 2^-27 has no integer solution with u < 2^24."""
    if F32(thresh) == F32(0.5):
        return ("eq", "exact", "up", "down", "band_above", "band_below")
    if integer_boxes and F32(thresh) == F32(0.2):
        return ("eq", "up", "down", "band_above", "band_below")
    return ("eq", "eq_above", "up", "down", "band_above", "band_below")


def iou_terms(a, b):
    """(inter, union, iou) in float32 exactly as oracle.postproc.iou_row and csrc/nms_iou.cuh evaluate them."""
    one = F32(1)
    w = max(F32(0), F32(F32(min(a[2], b[2]) - max(a[0], b[0])) + one))
    h = max(F32(0), F32(F32(min(a[3], b[3]) - max(a[1], b[1])) + one))
    inter = F32(w * h)
    sa = F32(F32(F32(a[2] - a[0]) + one) * F32(F32(a[3] - a[1]) + one))
    sb = F32(F32(F32(b[2] - b[0]) + one) * F32(F32(b[3] - b[1]) + one))
    u = F32(F32(sa + sb) - inter)
    return inter, u, F32(inter / u)


def classify(a, b, thresh):
    """Borderline classes of the pair (a, b) at T = float32(thresh), from the exact rationals of its float32 terms:
    eq          float32 IoU == T                         (not above: both boxes stay)
    eq_above    float32 IoU == T although inter / u > T  (a sign-of-(inter - T u) decision would suppress)
    exact       inter / u == T exactly
    up / down   float32 IoU == nextafter(T, +inf) / nextafter(T, -inf)
    band_above  0 < inter - T u <= 2^-20 max(inter, u)   (iou_above falls back to the division)
    band_below  -2^-20 max(inter, u) <= inter - T u < 0"""
    T = F32(thresh)
    inter, u, q = iou_terms(a, b)
    fi, fu, ft = Fraction(float(inter)), Fraction(float(u)), Fraction(float(T))
    d = fi - ft * fu
    inband = abs(d) <= BAND * max(fi, fu)
    out = set()
    if q == T:
        out.add("eq")
        if d > 0:
            out.add("eq_above")
    if d == 0:
        out.add("exact")
    if q == np.nextafter(T, F32(np.inf)):
        out.add("up")
    if q == np.nextafter(T, F32(-np.inf)):
        out.add("down")
    if inband and d > 0:
        out.add("band_above")
    if inband and d < 0:
        out.add("band_below")
    return out


PAIR_H = 16                      # rows of the column-pair map
PAIR_ANCHORS = (0, 1, 2, 3, 4)   # decoded box heights (+1 convention) at dh = 0: 13, 17, 25, 35, 49


def _column_pair_boxes(a, ra, dya, rb, dys):
    """Box A (anchor a at row ra, moved by dya) and the boxes B (anchor a at row rb, each dy of dys), decoded as the
    oracle does.  The column does not matter: every box spans its anchor's 17 columns."""
    anch = postproc.shifted_anchors(PAIR_H, 1)[[ra * 10 + a, rb * 10 + a]].astype(F32)
    d = np.zeros((len(dys) + 1, 4), F32)
    d[0, 1] = dya
    d[1:, 1] = dys
    boxes = postproc.decode_boxes(np.concatenate([anch[:1], np.repeat(anch[1:], len(dys), 0)]), d)
    return boxes[0], boxes[1:]


def column_pair_classes(a, ra, dya, rb, dyb, thresh):
    box_a, box_b = _column_pair_boxes(a, ra, dya, rb, np.array([dyb], F32))
    return classify(box_a, box_b[0], thresh)


def _column_pair_candidates(thresh, a, row, dya, steps=1500):
    """B one row below A, its dy stepped one float32 ulp at a time around the dy that puts IoU(A, B) on thresh.
    Yields (dy_b, decoded box B, classes) for the steps whose IoU lies within 4e-6 of thresh."""
    anch = postproc.shifted_anchors(PAIR_H, 1)[row * 10 + a]
    L = float(anch[3] - anch[1] + 2)                   # decoded box height (+1 convention)
    ov = 2 * L * thresh / (1 + thresh)                  # overlap rows that put ov / (2L - ov) on thresh
    shift = ov - (L - 16) - float(dya) * (L - 1)        # B's anchor sits 16 rows below A's
    dy0 = F32(-shift / (L - 1))
    dys = (np.array([dy0], F32).view(np.int32)[0] + np.arange(-steps, steps + 1, dtype=np.int32)).view(F32)
    box_a, box_b = _column_pair_boxes(a, row, dya, row + 1, dys)
    q = postproc.iou_row(box_a, box_b)
    for k in np.nonzero(np.abs(q.astype(np.float64) - float(F32(thresh))) < 4e-6)[0]:
        yield dys[k], tuple(box_a) + tuple(box_b[k]), classify(box_a, box_b[k], thresh)


def column_pairs(thresh, per_class=3):
    """Borderline pairs for the column NMS, [(anchor a, row of A, dy of A, row of B, dy of B, classes)], with at least
    per_class of every required class (a ValueError otherwise).  Besides the pairs found by stepping dy, two exact pairs:
    thresh 0.7: two 17-high boxes (anchor 1) overlapping 14 rows, IoU 14/20 = 0.7 > float32(0.7) with float32 quotient
                float32(0.7) -- the oracle keeps both;
    thresh 0.5: two 69-high boxes (anchor 5, dy = -9/4 moves B up 153 rows from 11 rows below) overlapping 46 rows,
                IoU 46/92 = 0.5 exactly."""
    need = required_classes(thresh)
    out, have, seen = [], {c: 0 for c in need}, set()

    def add(entry):
        out.append(entry)
        for c in entry[-1]:
            if c in have:
                have[c] += 1
    if F32(thresh) == F32(0.7):
        add((1, 1, F32(0), 2, F32(-13 / 16), column_pair_classes(1, 1, F32(0), 2, F32(-13 / 16), thresh)))
    if F32(thresh) == F32(0.5):
        for ra in (2, 3, 4):
            add((5, ra, F32(0), ra + 11, F32(-2.25), column_pair_classes(5, ra, F32(0), ra + 11, F32(-2.25), thresh)))
    for dya in (0, 1, -1, 2, -2, 3, -3):              # sub-pixel positions of A (multiples of 1/64 of its height)
        for a in PAIR_ANCHORS:
            for dy, boxes, cl in _column_pair_candidates(thresh, a, 1, F32(dya / 64)):
                if boxes not in seen and any(have.get(c, per_class) < per_class for c in cl):
                    seen.add(boxes)
                    add((a, 1, F32(dya / 64), 2, dy, cl))
            if all(v >= per_class for v in have.values()):
                return out
    raise ValueError("column pairs at %g: only %s" % (thresh, have))


def column_pair_heads(pairs):
    """One pair per column c: box A (anchor a, its row and dy, score 0.9 - c/1000) and box B (anchor a, its row and dy,
    score 0.5 - c/1000).  Every other box is made invalid (dh = -8 shrinks it below min_size), so each column's NMS
    decides exactly one pair.  Returns (cls, bbox, info, [(index of A, index of B)])."""
    H, W = PAIR_H, len(pairs)
    cls, bbox = exact_heads(H, W)
    bbox[..., 3::4] = F32(-8)
    idx = []
    for c, (a, ra, dya, rb, dyb, _) in enumerate(pairs):
        for row, d, s in ((ra, dya, F32(0.9 - c / 1000)), (rb, dyb, F32(0.5 - c / 1000))):
            bbox[0, row, c, 4 * a + 1] = d
            bbox[0, row, c, 4 * a + 3] = F32(0)
            cls[0, row, c, 2 * a + 1] = s
            cls[0, row, c, 2 * a] = F32(1) - s
        idx.append(((ra * W + c) * 10 + a, (rb * W + c) * 10 + a))
    info = np.array([[H * 16, W * 16, 1.0]], F32)
    return cls, bbox, info, idx


def generic_pair_boxes(wa, wb, ov, y=0):
    """Boxes A = [0, y, wa - 1, y] and B = [wa - ov, y, wa - ov + wb - 1, y]: height 1, so inter = ov, and the union is
    wa + wb - ov once float32 has rounded wa + wb (exact below 2^24)."""
    return np.array([0, y, wa - 1, y], F32), np.array([wa - ov, y, wa - ov + wb - 1, y], F32)


def generic_pairs(thresh, per_class=4):
    """Borderline pairs for the generic bitmask NMS, [(wa, wb, ov, classes)] (see generic_pair_boxes), with at least
    per_class of every required class; at 0.5 the exact ones have 3 ov = wa + wb."""
    T = Fraction(float(F32(thresh)))
    need = required_classes(thresh, integer_boxes=True)
    have = {c: 0 for c in need}
    out = []

    def add(wa, wb, ov):
        cl = classify(*generic_pair_boxes(wa, wb, ov), thresh)
        if any(have.get(c, per_class) < per_class for c in cl):
            out.append((wa, wb, ov, cl))
            for c in cl:
                if c in have:
                    have[c] += 1
    if F32(thresh) == F32(0.5):
        for ov in (7, 1000, 123457, 2796203):
            add(ov, 2 * ov, ov)
    # unions just below 2^24, and just below the largest one whose wa + wb = u + ov is still exact in float32
    top = int((2 ** 24 - 1) / (1 + thresh))
    for u in list(range(2 ** 24 - 1, 2 ** 24 - 8192, -1)) + list(range(top, top - 8192, -1)):
        base = T * u
        for ov in (base.numerator // base.denominator, base.numerator // base.denominator + 1):
            add((u + ov) // 2, u + ov - (u + ov) // 2, ov)
        if all(v >= per_class for v in have.values()):
            return out
    raise ValueError("generic pairs at %g: only %s" % (thresh, have))


def generic_pair_dets(pairs, n, lead=0):
    """n boxes in visiting order (scores strictly descending): `lead` single boxes, then the pairs (A, then B; cycled as
    needed), each pair on its own row y = 2k (rows two apart never overlap), then single boxes up to n.  lead = 1 puts
    pairs across the even 64-box block edges."""
    rows, y = [], 0
    for _ in range(lead):
        rows.append([0, y, 99, y])
        y += 2
    k = 0
    while len(rows) + 2 <= n:
        rows.extend(b.tolist() for b in generic_pair_boxes(*pairs[k % len(pairs)][:3], y=y))
        y += 2
        k += 1
    while len(rows) < n:
        rows.append([0, y, 99, y])
        y += 2
    dets = np.zeros((n, 5), F32)
    dets[:, :4] = np.asarray(rows, F32).reshape(-1, 4)
    dets[:, 4] = (1.0 - np.arange(n) / (2.0 * n)).astype(F32)
    return dets


# ---- whole-layer cases -----------------------------------------------------------------------------------------------
MIXED_HW = (62, 37)


def mixed_batch(nms_thresh=0.7):
    """Three images on the 62 x 37 map of a portrait blob: (0) structured; (1) im_info narrower than the map (300 px)
    with im_info[2] = 0.1, so the boxes of the columns past the edge are clipped to 1-px boxes that stay valid
    (min_size * 0.1 < 1) and start off their anchor column; (2) width 16 * 36 + 1 with im_info[2] = 0.1: only the last
    column is clipped, to a valid 1-px box that starts on its anchor, which trips the width trigger alone."""
    H, W = MIXED_HW
    cls, bbox = random_heads(300, 3, H, W)
    info = np.array([[H * 16, W * 16, 1.0], [H * 16, 300, 0.1], [H * 16, 16 * (W - 1) + 1, 0.1]], F32)
    return cls, bbox, info


RAGGED_EXTENTS = ((62, 37), (40, 30), (55, 20))


def column_census(cls, bbox, info, nms_thresh=0.7, **kw):
    """Per feature-map column of one image: the number of NMS candidates (no pre-NMS cut) and the positions, within the
    column's score order, of the boxes the oracle suppresses."""
    W = cls.shape[2]
    boxes, scores, order = sorted_candidates(cls, bbox, info, **kw)
    kept = set(postproc.nms_sorted(boxes, nms_thresh).tolist())
    col = (order // 10) % W
    count, suppressed = np.zeros(W, int), [[] for _ in range(W)]
    for r, c in enumerate(col):
        if r not in kept:
            suppressed[c].append(count[c])
        count[c] += 1
    return count, suppressed


# ---- comparison with the oracle --------------------------------------------------------------------------------------
LAYER_CFG = dict(RPN_PRE_NMS_TOP_N=12000, RPN_POST_NMS_TOP_N=1000, RPN_NMS_THRESH=0.7, RPN_MIN_SIZE=8, FEAT_STRIDE=16,
                 ANCHORS_PY2=False)      # ctpn_b200.engine.DEFAULT_CFG, the keys the proposal layer reads


def oracle_layer(cls, bbox, info, cfg=None):
    """postproc.proposal_layer of one image [1,H,W,..] under an Engine-style cfg: (blob [n,5], index [n])."""
    c = dict(LAYER_CFG, **(cfg or {}))
    blob, _, idx = postproc.proposal_layer(cls, bbox, info, c["RPN_PRE_NMS_TOP_N"], c["RPN_POST_NMS_TOP_N"],
                                           c["RPN_NMS_THRESH"], c["RPN_MIN_SIZE"], c["FEAT_STRIDE"], exp_mode="rounded",
                                           py2=bool(c["ANCHORS_PY2"]), return_index=True)
    return blob, idx


def layer_mismatches(rois, index, count, want_blob, want_idx):
    """Differences between one image's device rows (rois [rows,5], index [rows], count) and the oracle's: the first
    count rows bit for bit, every later row zero with index -1.  [] when they agree."""
    n, out = int(count), []
    if n != len(want_blob):
        return ["count %d, oracle %d" % (n, len(want_blob))]
    if not np.array_equal(np.asarray(index[:n]), want_idx):
        bad = np.nonzero(np.asarray(index[:n]) != want_idx)[0]
        out.append("index differs at %d rows, first at row %d: %s vs oracle %s"
                   % (len(bad), bad[0], index[bad[0]], want_idx[bad[0]]))
    if not np.array_equal(np.ascontiguousarray(rois[:n], F32).view(np.uint32), np.ascontiguousarray(want_blob, F32).view(np.uint32)):
        out.append("rois differ from the oracle's bits")
    if np.ascontiguousarray(rois[n:], F32).view(np.uint32).any() or (np.asarray(index[n:]) != -1).any():
        out.append("rows past count are not zero / -1")
    return out
