"""GPU: every path ctpn_proposals can dispatch -- column NMS in static and opt-in shared memory, up to 19 scan words,
the generic bitmask NMS for every image or per gated image, the bucketed and the gathered column lists -- and the generic
NMS entry points, bit for bit against the CPU oracle (oracle/postproc.py, exp_mode='rounded'), at the dispatch
boundaries (tests/proposal_cases.py restates the rule), on borderline IoU pairs, on sort ties and at config edges.
A launch census (torch.profiler kernel names) checks that the column kernel runs exactly when the rule says so."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import proposal_cases as P
from oracle import postproc

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32
COLUMN_KERNEL = "proposal_column_nms_kernel"
ALL = dict(RPN_PRE_NMS_TOP_N=-1, RPN_POST_NMS_TOP_N=-1)          # no pre- or post-NMS cut
NO_NMS = dict(ALL, RPN_NMS_THRESH=1.0)                            # IoU > 1 is impossible: every valid box, sorted


@pytest.fixture(scope="module")
def eng():
    from ctpn_b200.engine import Engine
    return Engine(None)


def launched_kernels(fn):
    """Names of the CUDA kernels fn() launches, from torch.profiler.  The profiler can come back without the kernel
    records of a capture (seen once on an H100); a capture that lacks the proposal layer's decode kernel is taken again,
    once, and must then have it."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for _ in range(2):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events()}
        if any("proposal_decode_kernel" in n for n in names):
            return out, names
    raise AssertionError("torch.profiler recorded no proposal_decode_kernel: %s" % sorted(names))


def run_layer(eng, cls, bbox, info, cfg=None, cls_is_logit=False, feat_sizes=None):
    """Engine.proposals: (rois, index, count) as numpy, and whether the column kernel ran."""
    import torch
    (rois, index, count), names = launched_kernels(lambda: eng.proposals(
        torch.from_numpy(cls).cuda(), torch.from_numpy(bbox).cuda(), torch.from_numpy(info), cls_is_logit=cls_is_logit,
        cfg=cfg, feat_sizes=feat_sizes))
    column = any(COLUMN_KERNEL in n for n in names)
    return rois.cpu().numpy(), index.cpu().numpy(), count.cpu().numpy(), column


def check_layer(eng, cls, bbox, info, cfg=None, path=None):
    """Every image of the batch against the oracle; path: the (nms, sort) pair the rule must give for this map, checked
    against the rule and, for column vs generic, against the kernels that ran."""
    c = dict(P.LAYER_CFG, **(cfg or {}))
    H, W = cls.shape[1:3]
    rule = P.dispatch(H, W, c["FEAT_STRIDE"])
    if path is not None:
        assert rule == path
    rois, index, count, column = run_layer(eng, cls, bbox, info, cfg)
    assert column == (rule[0] != "generic-all"), "column kernel ran: %s, rule: %s" % (column, rule)
    for b in range(cls.shape[0]):
        want, idx = P.oracle_layer(cls[b:b + 1], bbox[b:b + 1], info[b:b + 1], cfg)
        assert P.layer_mismatches(rois[b], index[b], count[b], want, idx) == [], "image %d" % b
    return rois, index, count


# (name, H, W, cfg, (nms path, sort path)) -- the name states the path; the rule and the census must agree with it
PATH_CASES = [
    ("column-static_51x20", 51, 20, {}, ("column-static", "bucketed")),
    ("column-optin_52x20", 52, 20, {}, ("column-optin", "bucketed")),
    ("column-optin_62x37_portrait", 62, 37, {}, ("column-optin", "bucketed")),
    ("column-optin_75x100_cfgB", 75, 100, {}, ("column-optin", "bucketed")),
    ("column-optin_19words_116x4", 116, 4, ALL, ("column-optin", "bucketed")),
    ("generic-all_117x4", 117, 4, {}, ("generic-all", None)),
    ("generic-all_stride8_37x56", 37, 56, dict(FEAT_STRIDE=8), ("generic-all", None)),
    ("column-static_stride32_20x30", 20, 30, dict(FEAT_STRIDE=32), ("column-static", "bucketed")),
    ("column-static_py2_30x40", 30, 40, dict(ANCHORS_PY2=True), ("column-static", "bucketed")),
    ("bucketed-last_6x256", 6, 256, {}, ("column-static", "bucketed")),
    ("gathered_6x257", 6, 257, {}, ("column-static", "gathered")),
]


@pytest.mark.parametrize("name,H,W,cfg,path", PATH_CASES, ids=[c[0] for c in PATH_CASES])
def test_dispatch_path_matches_oracle(eng, name, H, W, cfg, path):
    stride = cfg.get("FEAT_STRIDE", 16)
    cls, bbox = P.random_heads(H, 1, H, W)       # seed H: the 116-row case is the one tests/test_proposal_cases_cpu.py checks
    info = np.array([[H * stride, W * stride, 1.0]], F32)
    check_layer(eng, cls, bbox, info, cfg, path)


@pytest.mark.parametrize("thresh", [0.7, 0.03])
def test_mixed_batch_gates_images_to_the_generic_nms(eng, thresh):
    """One structured image, one whose clipped boxes start off their column, one with a valid 1-px column (the width
    trigger); at 0.03 every box trips the width trigger."""
    cls, bbox, info = P.mixed_batch()
    check_layer(eng, cls, bbox, info, dict(RPN_NMS_THRESH=thresh), ("column-optin", "bucketed"))


def test_ragged_canvas_matches_oracle_on_each_crop(eng):
    H, W = P.MIXED_HW
    cls, bbox = P.random_heads(400, 3, H, W)
    info = np.array([[h * 16, w * 16, 1.0] for h, w in P.RAGGED_EXTENTS], F32)
    rois, index, count, column = run_layer(eng, cls, bbox, info, feat_sizes=np.array(P.RAGGED_EXTENTS))
    assert column
    for b, (h, w) in enumerate(P.RAGGED_EXTENTS):
        want, idx = P.oracle_layer(np.ascontiguousarray(cls[b:b + 1, :h, :w]), np.ascontiguousarray(bbox[b:b + 1, :h, :w]), info[b:b + 1])
        assert P.layer_mismatches(rois[b], index[b], count[b], want, idx) == [], "image %d" % b


@pytest.mark.parametrize("thresh", [0.7, 0.5])
def test_borderline_column_pairs(eng, thresh):
    pairs = P.column_pairs(thresh)
    cls, bbox, info, idx = P.column_pair_heads(pairs)
    rois, index, count = check_layer(eng, cls, bbox, info, dict(RPN_NMS_THRESH=thresh), ("column-static", "bucketed"))
    kept = set(index[0, :count[0]].tolist())
    boxes = P.decoded(cls, bbox, info)[0]
    for (i, j), p in zip(idx, pairs):
        assert i in kept and (j in kept) == (P.iou_terms(boxes[i], boxes[j])[2] <= F32(thresh)), p


def _nms_host(dets, thresh):
    from ctpn_b200 import _native as N
    dets = np.ascontiguousarray(dets, F32)
    keep = np.zeros(len(dets), np.int32)
    num = C.c_int(0)
    N.check(N.lib.ctpn_nms_host(keep.ctypes.data, C.byref(num), dets.ctypes.data, len(dets), 5, F32(thresh), 0), "ctpn_nms_host")
    return keep[:num.value]


@pytest.mark.parametrize("thresh", [0.7, 0.5, 0.3, 0.2])
def test_borderline_generic_pairs_host(thresh):
    pairs = P.generic_pairs(thresh)
    for n in (64, 65, 128, 129):
        for lead in (0, 1):
            dets = P.generic_pair_dets(pairs, n, lead)
            np.testing.assert_array_equal(_nms_host(dets, thresh), postproc.nms_sorted(dets, thresh), err_msg="n=%d lead=%d" % (n, lead))


@pytest.mark.parametrize("thresh", [0.7, 0.3])
def test_borderline_generic_pairs_sorted_batched(thresh):
    """ctpn_nms_sorted, batch of 3 with ragged counts; max_keep unlimited, or ending exactly on the last box of the first
    or second 64-box block of image 0."""
    import torch
    from ctpn_b200 import _native as N
    pairs = P.generic_pairs(thresh)
    max_n, counts, leads = 200, [129, 64, 65], [1, 0, 1]
    imgs = [P.generic_pair_dets(pairs, c, lead) for c, lead in zip(counts, leads)]
    full0 = postproc.nms_sorted(imgs[0], thresh)
    edges = []
    for edge in (63, 127):
        m = int((full0 <= edge).sum())
        assert full0[m - 1] == edge
        edges.append(m)
    boxes = np.zeros((3, max_n, 4), F32)
    for b, d in enumerate(imgs):
        boxes[b, :len(d)] = d[:, :4]
    dev = torch.device("cuda", 0)
    bt, ct = torch.from_numpy(boxes).to(dev), torch.tensor(counts, dtype=torch.int32, device=dev)
    ws = torch.empty(N.lib.ctpn_nms_workspace_bytes(3, max_n), dtype=torch.uint8, device=dev)
    for max_keep in [0] + edges:
        stride = max_keep if max_keep > 0 else max_n
        keep = torch.full((3, stride), -1, dtype=torch.int32, device=dev)
        num = torch.zeros(3, dtype=torch.int32, device=dev)
        N.check(N.lib.ctpn_nms_sorted(N.ptr(bt), N.ptr(ct), 3, max_n, F32(thresh), max_keep, N.ptr(keep), N.ptr(num), N.ptr(ws),
                                      ws.numel(), N.stream_ptr()), "ctpn_nms_sorted")
        torch.cuda.synchronize()
        for b in range(3):
            want = postproc.nms_sorted(imgs[b], thresh, max_keep=max_keep)
            assert int(num[b]) == len(want), (max_keep, b)
            np.testing.assert_array_equal(keep[b, :len(want)].cpu().numpy(), want)


def _assert_sorted_rows(rois, index, n, scores_of):
    """Rows 0..n-1 in score order, ties by ascending anchor index; scores_of: the device score of every index."""
    s, i = rois[:n, 0], index[:n]
    np.testing.assert_array_equal(s.view(np.uint32), scores_of[i].view(np.uint32))
    ok = (s[:-1] > s[1:]) | ((s[:-1] == s[1:]) & (i[:-1] < i[1:]))
    assert ok.all(), "order broken at row %d" % np.nonzero(~ok)[0][0]


def softmax64(logits):
    l = logits.reshape(-1, 2).astype(np.float64)
    e = np.exp(l - l.max(1, keepdims=True))
    return e[:, 1] / e.sum(1)


def ulp_error(got, p):
    return np.abs(got.astype(np.float64) - p) / np.spacing(np.abs(p).astype(F32)).astype(np.float64)


def assert_softmax_within_4ulp(got, logits, idx, what):
    """Device probabilities within 4 float32 ulp of a float64 softmax of the float32 logit differences the kernel (like
    the reference's float32 softmax) forms, l - max(l0, l1).  That rounding alone moves exp(l1 - l0) by up to
    |l1 - l0| * 2^-24 relative, so against the exact logits the error grows with the difference; both maxima are
    printed.  Results below float32's normal range may also be flushed to 0."""
    l = logits.reshape(-1, 2)[idx]
    m = np.maximum(l[:, 0], l[:, 1])
    d = np.stack([l[:, 0] - m, l[:, 1] - m], 1).astype(np.float64)       # float32 subtraction, then exact
    e = np.exp(d)
    p = e[:, 1] / e.sum(1)
    err = ulp_error(got, p)
    flushed = (got == 0) & (p < np.finfo(F32).tiny)
    print("%s: device softmax max error %.3f ulp over %d probabilities (%d flushed to 0); %.3f ulp against the exact logits"
          % (what, err[~flushed].max(), len(p), flushed.sum(), ulp_error(got, softmax64(logits)[idx])[~flushed].max()))
    assert (err[~flushed] <= 4).all(), np.nonzero(err > 4)[0][:8]


def test_full_sort_order_logits_75x100(eng):
    """75 000 anchors (more than 65 536 keys, not a multiple of 1024), no suppression: every valid box comes back in
    decode + clip + filter + order_desc order, with its box bit for bit; every probability within 4 ulp of float64."""
    import torch
    H, W = 75, 100
    rs = np.random.RandomState(5)
    logits = (rs.standard_normal((1, H, W, 20)) * 2).astype(F32)
    bbox = (rs.standard_normal((1, H, W, 40)) * 0.3).astype(F32)
    info = np.array([[H * 16, W * 16, 1.0]], F32)
    rois, index, count = eng.proposals(torch.from_numpy(logits).cuda(), torch.from_numpy(bbox).cuda(), torch.from_numpy(info),
                                       cls_is_logit=True, cfg=NO_NMS)
    rois, index, n = rois[0].cpu().numpy(), index[0].cpu().numpy(), int(count[0])
    boxes, _, valid = P.decoded(np.zeros_like(logits), bbox, info)
    assert n == valid.sum() > 65536 and (H * W * 10) % 1024 != 0
    assert sorted(index[:n].tolist()) == np.nonzero(valid)[0].tolist()
    np.testing.assert_array_equal(rois[:n, 1:].view(np.uint32), boxes[index[:n]].view(np.uint32))
    scores_of = np.zeros(H * W * 10, F32)
    scores_of[index[:n]] = rois[:n, 0]
    _assert_sorted_rows(rois, index, n, scores_of)
    assert_softmax_within_4ulp(rois[:n, 0], logits, index[:n], "75x100 logits")


def test_full_sort_order_ties_and_ulp_pairs(eng):
    cls, bbox, pairs = P.ulp_pair_heads(75, 100)
    info = np.array([[1200, 1600, 1.0]], F32)
    rois, index, count, _ = run_layer(eng, cls, bbox, info, NO_NMS)
    boxes, scores, order = P.sorted_candidates(cls, bbox, info)
    n = int(count[0])
    assert n == len(order)
    np.testing.assert_array_equal(index[0, :n], order)
    np.testing.assert_array_equal(rois[0, :n, 0].view(np.uint32), scores.view(np.uint32))
    np.testing.assert_array_equal(rois[0, :n, 1:].view(np.uint32), boxes.view(np.uint32))
    pos = np.empty(cls.size // 2, np.int64)
    pos[order] = np.arange(n)
    assert (pos[pairs[:, 1]] < pos[pairs[:, 0]]).all()               # the higher score (larger index) first


def test_full_sort_order_equal_scores_cut_inside_tie_group(eng):
    H, W = 20, 30
    cls, bbox = P.random_heads(77, 1, H, W)
    cls[..., 1::2] = F32(0.5)
    info = np.array([[H * 16, W * 16, 1.0]], F32)
    cfg = dict(NO_NMS, RPN_PRE_NMS_TOP_N=1000)
    rois, index, count, _ = run_layer(eng, cls, bbox, info, cfg)
    boxes, scores, order = P.sorted_candidates(cls, bbox, info, pre=1000)
    assert int(count[0]) == 1000 == len(order)
    np.testing.assert_array_equal(index[0, :1000], order)
    np.testing.assert_array_equal(rois[0, :1000, 1:].view(np.uint32), boxes.view(np.uint32))


def test_signed_zero_scores_tie(eng):
    """-0.0 and +0.0 probabilities compare equal in the oracle's stable sort, so they come back by ascending index."""
    H, W = 6, 5
    cls, bbox = P.exact_heads(H, W)
    fg = cls[0, ..., 1::2].reshape(-1)
    fg[:] = F32(0.25)
    fg[[3, 10, 17, 40]] = F32(-0.0)
    fg[[4, 9, 16, 41]] = F32(0.0)
    cls[0, ..., 1::2] = fg.reshape(H, W, 10)
    info = np.array([[H * 16, W * 16, 1.0]], F32)
    rois, index, count = check_layer(eng, cls, bbox, info, NO_NMS)
    n = int(count[0])
    np.testing.assert_array_equal(index[0, n - 8:n], [3, 4, 9, 10, 16, 17, 40, 41])


def test_softmax_extremes(eng):
    pairs = [(0, 0), (3.5, 3.5), (-7, -7), (100, 0), (0, 100), (-100, 0), (0, -100), (1e30, -1e30), (-1e30, 1e30),
             (1e30, 1e30), (0.5, -0.25), (20, -20), (-88, 0), (0, 88)]
    H, W = 1, 2
    logits = np.zeros((1, H, W, 20), F32)
    flat = logits.reshape(-1, 2)
    flat[:len(pairs)] = np.asarray(pairs, F32)
    _, bbox = P.exact_heads(H, W)
    info = np.array([[H * 16 + 200, W * 16, 1.0]], F32)
    import torch
    rois, index, count = eng.proposals(torch.from_numpy(logits).cuda(), torch.from_numpy(bbox).cuda(), torch.from_numpy(info),
                                       cls_is_logit=True, cfg=NO_NMS)
    n = int(count[0])
    rois, index = rois[0, :n].cpu().numpy(), index[0, :n].cpu().numpy()
    got = np.zeros(H * W * 10, F32)
    got[index] = rois[:, 0]
    assert n == H * W * 10
    assert got[0] == 0.5 and got[1] == 0.5 and got[2] == 0.5
    assert got[4] == 1.0 and got[8] == 1.0 and got[7] == 0.0
    assert_softmax_within_4ulp(got, logits, np.arange(H * W * 10), "extremes")


def test_min_size_boundary_keeps_boxes_equal_to_it(eng):
    """dh = 0: anchor 0's boxes are exactly 13 rows high (+1 convention); RPN_MIN_SIZE = 13 keeps them (>=).  No NMS, so
    that every valid box comes back."""
    H, W = 6, 5
    cls, bbox = P.random_heads(31, 1, H, W)
    bbox[:] = 0
    info = np.array([[H * 16 + 300, W * 16, 1.0]], F32)
    _, index, count = check_layer(eng, cls, bbox, info, dict(NO_NMS, RPN_MIN_SIZE=13))
    assert int((index[0, :count[0]] % 10 == 0).sum()) == H * W
    _, index, count = check_layer(eng, cls, bbox, info, dict(NO_NMS, RPN_MIN_SIZE=13.5))
    assert int((index[0, :count[0]] % 10 == 0).sum()) == 0


def test_no_valid_box(eng):
    cls, bbox = P.random_heads(32, 2, 12, 18)
    info = np.array([[192, 288, 1.0]] * 2, F32)
    rois, index, count = check_layer(eng, cls, bbox, info, dict(RPN_MIN_SIZE=2000))
    assert (count == 0).all() and not rois.any() and (index == -1).all()


def test_fewer_valid_boxes_than_pre(eng):
    cls, bbox = P.random_heads(33, 1, 12, 18)
    info = np.array([[192, 288, 1.0]], F32)
    cfg = dict(RPN_MIN_SIZE=16, RPN_PRE_NMS_TOP_N=2000, RPN_POST_NMS_TOP_N=-1)      # 2000 < 2160 anchors
    assert P.decoded(cls, bbox, info, min_size=16)[2].sum() < 2000
    check_layer(eng, cls, bbox, info, cfg)


def test_post_larger_than_pre(eng):
    cls, bbox = P.random_heads(34, 1, 20, 30)
    info = np.array([[320, 480, 1.0]], F32)
    rois, index, count = check_layer(eng, cls, bbox, info, dict(RPN_PRE_NMS_TOP_N=500, RPN_POST_NMS_TOP_N=800))
    assert rois.shape == (1, 800, 5) and 0 < count[0] <= 500
    assert not rois[0, 500:].any() and (index[0, 500:] == -1).all()


def test_undersized_workspace_fails_before_any_launch():
    import torch
    from ctpn_b200 import _native as N
    H, W = 12, 18
    cls, bbox = (torch.from_numpy(x).cuda() for x in P.random_heads(35, 1, H, W))
    info = torch.tensor([[192, 288, 1.0]], device="cuda")
    need = N.lib.ctpn_proposals_workspace_bytes(1, H, W, 12000)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    rois = torch.full((1, 1000, 5), 7.0, device="cuda")
    index = torch.full((1, 1000), 7, dtype=torch.int32, device="cuda")
    count = torch.full((1,), 7, dtype=torch.int32, device="cuda")
    rc = N.lib.ctpn_proposals(N.ptr(cls), 0, N.ptr(bbox), N.ptr(info), 1, H, W, 16, 12000, 1000, 0.7, 8.0, 0, N.ptr(rois),
                              N.ptr(index), N.ptr(count), N.ptr(ws), need - 1, N.stream_ptr())
    torch.cuda.synchronize()
    assert rc == N.ERR_WORKSPACE and "workspace" in N.last_error()
    assert (rois == 7).all() and (index == 7).all() and int(count[0]) == 7


def run_proposal_check(cmd, switch):
    env = dict(os.environ, CTPN_B200_LIB="dbg", **{switch: "1"})
    p = subprocess.run([sys.executable, os.path.join(HERE, "proposal_checks.py"), cmd], capture_output=True, text=True,
                       timeout=600, env=env)
    lines = [l for l in p.stdout.strip().splitlines() if l.startswith("{")]
    assert lines, "no result line.\nstdout:\n%s\nstderr:\n%s" % (p.stdout[-2000:], p.stderr[-3000:])
    res = json.loads(lines[-1])
    print(cmd, switch, "->", json.dumps(res))
    assert res["ok"] and p.returncode == 0, "%s\nstderr:\n%s" % (json.dumps(res), p.stderr[-2000:])


@pytest.mark.parametrize("cmd,switch", [("mixed", "CTPN_COLUMN_GATHER"), ("column_pairs", "CTPN_COLUMN_GATHER"),
                                        ("column_pairs", "CTPN_GENERIC_NMS")])
def test_test_library_switches(cmd, switch):
    run_proposal_check(cmd, switch)
