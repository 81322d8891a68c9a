"""GPU: the whole engine against the CPU oracle (oracle/net_cpu.py + oracle/postproc.py) on the same
seeded synthetic weights and images: layer-by-layer activations, head tensors, proposals through
the reference-named API (get_network / Session / test_ctpn), batching, and the SIMT-vs-tensor-core
cross-check.  Floating-point tolerance: north_star's 1e-3, judged as |a-b| <= 1e-3*max(1,|b|);
the tighter per-mode bounds asserted here are the measured behaviour of each plane count."""
import numpy as np
import pytest
import torch

from oracle import net_cpu, postproc, synth

pytestmark = pytest.mark.gpu

TAPS = ["conv1_1", "conv1_2+pool", "conv2_1", "conv2_2+pool", "conv3_3+pool", "conv4_3+pool", "conv5_3",
        "rpn_conv/3x3", "lstm_out", "lstm_o"]


@pytest.fixture(scope="module")
def weights():
    return synth.make_weights(0)


def rel_err(got, want):
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-12))


@pytest.mark.parametrize("planes,tol", [(3, 5e-4), (2, 5e-4), (4, 5e-4), (1, 1.5e-1)])
def test_layerwise_against_float64_oracle(weights, planes, tol):
    from ctpn_b200 import Engine
    im = synth.make_image(7, 96, 160)                      # feature map 6 x 10
    blob = (im.astype(np.float32) - net_cpu.PIXEL_MEANS.astype(np.float64)).astype(np.float32)[None]
    ref = net_cpu.forward(blob, weights, dtype=torch.float64, taps=TAPS)
    eng = Engine(weights, planes=planes, keep_activations=True)
    cls, bbox = eng.forward_heads(torch.from_numpy(im[None]).cuda())
    torch.cuda.synchronize()
    worst = {}
    for name in TAPS:
        want = ref[name]
        got = eng.tap(name).cpu().numpy().reshape(want.shape)
        worst[name] = rel_err(got, want)
    worst["rpn_cls_score"] = rel_err(cls.cpu().numpy(), ref["rpn_cls_score"])
    worst["rpn_bbox_pred"] = rel_err(bbox.cpu().numpy(), ref["rpn_bbox_pred"])
    print(planes, {k: "%.2e" % v for k, v in worst.items()})
    assert max(worst.values()) < tol, worst


def test_uint8_and_float_blob_inputs_agree_bitwise(weights):
    """Feeding uint8 pixels (mean subtraction fused in conv1_1) == feeding the reference's float32 blob."""
    from ctpn_b200 import Engine
    eng = Engine(weights, planes=2)
    im = synth.make_image(3, 64, 80)
    blob = im.astype(np.float32)
    blob -= net_cpu.PIXEL_MEANS                              # numpy semantics of test.py:9
    a = eng.forward_heads(torch.from_numpy(im[None]).cuda())
    b = eng.forward_heads(torch.from_numpy(blob[None]).cuda())
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def _match_rois(got, got_idx, want, want_idx):
    """Compare two roi sets by anchor index; returns (fraction of reference rows found, max score diff,
    max box diff relative to max(1,|b|))."""
    pos = {int(i): k for k, i in enumerate(got_idx)}
    common = [(pos[int(i)], k) for k, i in enumerate(want_idx) if int(i) in pos]
    if not common:
        return 0.0, np.inf, np.inf
    g = got[[c[0] for c in common]]
    w = want[[c[1] for c in common]]
    ds = np.abs(g[:, 0] - w[:, 0]).max()
    db = (np.abs(g[:, 1:] - w[:, 1:]) / np.maximum(1.0, np.abs(w[:, 1:]))).max()
    return len(common) / float(len(want_idx)), float(ds), float(db)


def rows_matched(got, want, tol=1e-3):
    """Fraction of the oracle's rows (score, x1, y1, x2, y2) for which the engine has a row within tol * max(1, |b|)."""
    if not len(want):
        return 1.0
    hit = 0
    for r in want:
        hit += bool(len(got)) and bool((np.abs(got - r).max(axis=1) <= tol * max(1.0, float(np.abs(r).max()))).any())
    return hit / float(len(want))


# head max|diff| cls / bbox vs the float32 oracle at 600x900, per arithmetic (planes 2 = bf16x2, 3 = bf16x3, 4 = f16f8):
# bounds with headroom over the measured deviations, all inside 1e-3
HEAD_BOUNDS = {2: (6e-4, 8e-5), 3: (4e-4, 6e-5), 4: (1e-3, 2e-4)}


@pytest.mark.parametrize("planes", [2, 3, 4])
def test_end_to_end_600x900_against_oracle(weights, planes):
    """BASELINE.json config 1/2 shape: one 600x900 image, full path.  Head tensors within 1e-3;
    proposals: bit-exact against the oracle when both start from the engine's head tensors, and
    >= 99.9% identical rows (scores within 1e-5, boxes within 2e-4 relative) against the all-CPU oracle path."""
    from ctpn_b200 import Engine
    eng = Engine(weights, planes=planes)
    im = synth.make_image(0)
    blob, scale = net_cpu.image_blob(im)
    assert scale == 1.0
    ref = net_cpu.forward(blob, weights)                    # float32 oracle
    cls, bbox = eng.forward_heads(torch.from_numpy(im[None]).cuda())
    cls_h, bbox_h = cls.cpu().numpy(), bbox.cpu().numpy()
    d_cls, d_box = np.abs(cls_h - ref["rpn_cls_score"]).max(), np.abs(bbox_h - ref["rpn_bbox_pred"]).max()
    print("planes", planes, "head max|diff| vs float32 oracle: cls %.2e bbox %.2e" % (d_cls, d_box))
    assert d_cls < HEAD_BOUNDS[planes][0] and d_box < HEAD_BOUNDS[planes][1]
    info = np.array([[600, 900, 1.0]], np.float32)
    rois, index, count = eng.proposals(cls, bbox, torch.from_numpy(info), cls_is_logit=True)
    n = int(count[0])
    got, got_idx = rois[0, :n].cpu().numpy(), index[0, :n].cpu().numpy()
    # (1) same head tensors in -> identical rows out (index work is bit-exact)
    # oracle-side softmax of the engine's logits (may differ from the device's expf in the last ulp, hence
    # 99.5% instead of 100% row identity)
    l = cls_h.reshape(-1, 2).astype(np.float64)
    e = np.exp(l - l.max(1, keepdims=True))
    prob = (e / e.sum(1, keepdims=True)).astype(np.float32).reshape(cls_h.shape)
    want, _, want_idx = postproc.proposal_layer(prob, bbox_h, info, return_index=True)
    frac, ds, db = _match_rois(got, got_idx, want, want_idx)
    assert frac >= 0.995 and ds < 1e-6 and db < 1e-6, (frac, ds, db)
    # (2) all-CPU oracle path
    want2, _, want2_idx = postproc.proposal_layer(ref["rpn_cls_prob_reshape"], ref["rpn_bbox_pred"], info, return_index=True)
    frac, ds, db = _match_rois(got, got_idx, want2, want2_idx)
    print("planes", planes, "e2e overlap %.4f  dscore %.2e  dbox %.2e" % (frac, ds, db))
    assert frac >= 0.999 and ds < 1e-5 and db < 2e-4, (frac, ds, db)


def test_reference_api_test_ctpn_and_text_detector(weights):
    """The reference call sequence (demo.py:79-105 / test.py:40-58) on the stand-in Session, for an
    image that needs no rescale (uint8 fast path) and one that does (float32 blob path)."""
    from ctpn_b200 import Session
    from lib.fast_rcnn.config import cfg
    from lib.fast_rcnn.test import test_ctpn
    from lib.networks.factory import get_network
    from lib.text_connector.detectors import TextDetector
    sess = Session(weights, planes=2)
    net = get_network("VGGnet_test")
    with pytest.raises(KeyError):
        get_network("ResNet_test")
    for seed, (h, w) in [(1, (600, 900)), (2, (300, 400))]:
        im = synth.make_image(seed, h, w)
        scores, boxes = test_ctpn(sess, net, im)
        blob, scale = net_cpu.image_blob(im)
        ref = net_cpu.forward(blob, weights)
        info = np.array([[blob.shape[1], blob.shape[2], scale]], np.float32)
        want, _ = postproc.proposal_layer(ref["rpn_cls_prob_reshape"], ref["rpn_bbox_pred"], info)
        assert scores.dtype == np.float32 and boxes.shape == (scores.shape[0], 4)
        assert (np.diff(scores) <= 0).all() and scores.shape[0] <= cfg.TEST.RPN_POST_NMS_TOP_N
        # ALL rows: same count up to NMS decisions that sit within float noise of the threshold, every oracle row present
        assert abs(scores.shape[0] - want.shape[0]) <= 2
        got = np.hstack([scores[:, None], boxes * np.float32(scale)])
        assert rows_matched(got, want) >= 0.995
        lines = TextDetector().detect(boxes, scores[:, np.newaxis], im.shape[:2])
        assert lines.ndim == 2 and lines.shape[1] == 9 and lines.dtype == np.float64


@pytest.mark.parametrize("h,w,n", [(128, 192, 3), (600, 900, 2), (300, 300, 5)])
def test_f16f8_batch_equals_singles_row_stacked_maps(weights, h, w, n):
    """F16F8 mode stores the 1/16-scale maps of a batch row-stacked (one tall image with zero pad rows, fewer 16-row tiles);
    a single image is not stacked.  Same calibrated scales -> the batched results must equal the per-image ones bit for bit."""
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="f16f8")
    ims = np.stack([synth.make_image(80 + i, h, w) for i in range(n)])
    batch = eng.detect_batch(ims)                 # first call: calibrates the activation scales on this batch
    cls_b, box_b = eng.forward_heads(torch.from_numpy(ims).cuda())
    for i in range(n):
        s, b = eng.detect(ims[i])
        np.testing.assert_array_equal(s, batch[i][0])
        np.testing.assert_array_equal(b, batch[i][1])
        c1, b1 = eng.forward_heads(torch.from_numpy(ims[i:i + 1]).cuda())
        assert torch.equal(c1[0], cls_b[i]) and torch.equal(b1[0], box_b[i])


def test_streaming_api_with_large_distinct_unpinned_batches(weights):
    """ADVICE r1: rois_batches stages ndarray / unpinned batches through pinned buffers while the previous batch's H2D may
    still be in flight.  Four distinct 13 MB ndarray batches (H2D ~ 1 ms each): every streamed result must equal the
    one-batch-at-a-time result, i.e. no batch may see pixels of its successor."""
    from ctpn_b200 import Engine
    eng = Engine(weights, planes=1)
    rs = np.random.RandomState(5)
    batches = [rs.randint(0, 256, size=(8, 600, 900, 3), dtype=np.uint8) for _ in range(4)]
    want = [eng.rois_batch(b) for b in batches]
    got = list(eng.rois_batches(iter(batches)))
    got_again = list(eng.rois_batches(torch.from_numpy(b) for b in batches))      # unpinned CPU tensors take the same route
    assert len(got) == len(got_again) == 4
    for k in range(4):
        for i in range(8):
            np.testing.assert_array_equal(got[k][i], want[k][i])
            np.testing.assert_array_equal(got_again[k][i], want[k][i])


def test_f16f8_recalibration_and_graph_invalidation(weights):
    """F16F8 activation scales are frozen after the first batch; recalibrate() re-derives them from the next one and drops the
    captured CUDA graphs (they hold the old scales as kernel arguments): an engine calibrated on a flat grey image (the demo's
    warm-up) and then recalibrated must give exactly what a fresh engine gives on that image."""
    from ctpn_b200 import Engine
    grey = 128 * np.ones((300, 300, 3), np.uint8)
    im = synth.make_image(33, 300, 300)
    eng = Engine(weights, mode="f16f8")
    for _ in range(4):                              # warm-up as ctpn/demo.py: calibrates on the grey image, captures a graph
        eng.detect(grey)
    stale = eng.detect(im)[0]
    eng.recalibrate()
    assert not eng._graphs
    got = [eng.detect(im) for _ in range(4)]        # eager, eager, capture + replay, replay
    want = Engine(weights, mode="f16f8").detect(im)
    for s_, b_ in got:
        np.testing.assert_array_equal(s_, want[0])
        np.testing.assert_array_equal(b_, want[1])
    print("scores with scales from the grey image differ from the recalibrated ones by %.2e" % float(np.abs(stale[:50] - want[0][:50]).max()))


def test_small_batches_replay_a_cuda_graph_per_shape_bucket(weights):
    """Batches of <= graph_max_batch images run as a CUDA graph captured on the third call of a (shape, dtype) bucket; the
    replayed results must equal the eager ones bit for bit, also when two buckets alternate and inputs change between calls."""
    from ctpn_b200 import Engine
    eager = Engine(weights, planes=2, graph_max_batch=0)
    eng = Engine(weights, planes=2)
    a = [synth.make_image(90 + i, 96, 160) for i in range(4)]
    b = [synth.make_image(95 + i, 160, 96) for i in range(4)]
    for rnd in range(4):                                    # calls 1-2 eager, 3 captures + replays, 4 replays
        for im in (a[rnd], b[rnd]):
            s0, b0 = eager.detect(im)
            s1, b1 = eng.detect(im)
            np.testing.assert_array_equal(s1, s0)
            np.testing.assert_array_equal(b1, b0)
    assert sum("graph" in g for g in eng._graphs.values()) == 2
    pair = np.stack(a[:2])                                  # batch 2 is its own bucket
    for _ in range(4):
        got = eng.detect_batch(pair)
        want = eager.detect_batch(pair)
        for g, w_ in zip(got, want):
            np.testing.assert_array_equal(g[0], w_[0])


def test_demo_pb_frozen_graph_path_equals_checkpoint_path(weights, tmp_path, monkeypatch):
    """ctpn/demo_pb.py (demo_pb.py:55-98 of the reference): weights from a frozen GraphDef, head tensors fetched by graph name,
    proposal_layer called directly, TextDetector, res file -- the same result file as ctpn/demo.py's ctpn() on that image."""
    import cv2
    import tf_format_writer as W
    from ctpn import demo, demo_pb
    from ctpn_b200 import Session
    from lib.networks.factory import get_network
    pb = str(tmp_path / "ctpn.pb")
    W.write_frozen_graph(pb, weights)
    im_path = str(tmp_path / "img_7.png")
    cv2.imwrite(im_path, synth.make_image(70, 450, 640))
    out_a, out_b = tmp_path / "a", tmp_path / "b"
    out_a.mkdir(); out_b.mkdir()
    sess = Session(planes=2)
    sess.restore(pb)
    with pytest.raises(KeyError):
        sess.graph.get_tensor_by_name("conv5_3/Relu:0")
    monkeypatch.setattr(demo, "RESULTS_DIR", str(out_a))
    lines = demo_pb.detect_pb(sess, im_path)
    assert lines.ndim == 2 and lines.shape[1] == 9
    monkeypatch.setattr(demo, "RESULTS_DIR", str(out_b))
    demo.ctpn(Session(weights, planes=2), get_network("VGGnet_test"), im_path)
    assert open(out_a / "res_img_7.txt", "rb").read() == open(out_b / "res_img_7.txt", "rb").read()


def test_batch_equals_singles_and_simt_cross_check(weights):
    from ctpn_b200 import Engine
    eng = Engine(weights, planes=2)
    ims = np.stack([synth.make_image(20 + i, 128, 192) for i in range(3)])
    batch = eng.detect_batch(ims)
    for i in range(3):
        s, b = eng.detect(ims[i])
        np.testing.assert_array_equal(s, batch[i][0])
        np.testing.assert_array_equal(b, batch[i][1])
    streamed = list(eng.rois_batches([ims, ims[::-1].copy()]))          # pipelined API == per-batch API
    for i in range(3):
        np.testing.assert_array_equal(streamed[0][i][:, 0], batch[i][0])
        np.testing.assert_array_equal(streamed[1][2 - i][:, 0], batch[i][0])
    # float32 SIMT convolutions (test library, own process), same planes: head tensors within 5e-4
    from test_conv_gpu import DBG, run_check
    run_check("net_simt", "--B", 3, "--H", 128, "--W", 192, "--planes", 2, "--tol", 5e-4, env=DBG)


def test_bf16_mode_measured_deviation(weights):
    """BASELINE.json configs[2] arithmetic (bf16 operands, planes=1) does NOT meet the 1e-3 bar; this pins what it does
    deliver at 600x900."""
    from ctpn_b200 import Engine
    eng = Engine(weights, planes=1)
    im = synth.make_image(7)
    blob, _ = net_cpu.image_blob(im)
    ref = net_cpu.forward(blob, weights)
    info = np.array([[600, 900, 1.0]], np.float32)
    want, _ = postproc.proposal_layer(ref["rpn_cls_prob_reshape"], ref["rpn_bbox_pred"], info)
    cls, bbox = eng.forward_heads(torch.from_numpy(im[None]).cuda())
    d_cls = np.abs(cls.cpu().numpy() - ref["rpn_cls_score"]).max()
    d_box = np.abs(bbox.cpu().numpy() - ref["rpn_bbox_pred"]).max()
    frac = rows_matched(eng.rois_batch(im[None], info)[0], want)
    print("bf16: head cls %.3e bbox %.3e, oracle rows matched %.3f" % (d_cls, d_box, frac))
    assert d_cls < 0.25 and d_box < 0.05 and frac >= 0.90


@pytest.mark.parametrize("seed", [11, 12, 13, 14, 15, 16])
def test_f16f8_mode_head_error_over_several_images(weights, seed):
    """The 2-unit arithmetic on more images than the one of test_end_to_end: every one must stay inside the 1e-3 contract on
    the head tensors with all oracle rows reproduced."""
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="f16f8")
    im = synth.make_image(seed)
    blob, _ = net_cpu.image_blob(im)
    ref = net_cpu.forward(blob, weights)
    info = np.array([[600, 900, 1.0]], np.float32)
    want, _ = postproc.proposal_layer(ref["rpn_cls_prob_reshape"], ref["rpn_bbox_pred"], info)
    cls, bbox = eng.forward_heads(torch.from_numpy(im[None]).cuda())
    d_cls = np.abs(cls.cpu().numpy() - ref["rpn_cls_score"]).max()
    d_box = np.abs(bbox.cpu().numpy() - ref["rpn_bbox_pred"]).max()
    frac = rows_matched(eng.rois_batch(im[None], info)[0], want)
    print("f16f8 seed %d: head cls %.3e bbox %.3e, oracle rows matched %.4f" % (seed, d_cls, d_box, frac))
    assert d_cls < 1e-3 and d_box < 2e-4 and frac >= 0.995


def test_config4_high_resolution_1200x1600(weights):
    """BASELINE.json configs[3]: 1200x1600 images (75x100 feature map, 75 000 anchors, 12 000 into NMS).
    Uses the engine API directly (the reference's test_ctpn would first shrink the image to 600x800 unless
    cfg.TEST.SCALES / MAX_SIZE are overridden, SURVEY.md 8d)."""
    from ctpn_b200 import Engine
    eng = Engine(weights, planes=2)
    ims = np.stack([synth.make_image(40 + i, 1200, 1600) for i in range(2)])
    info = np.array([[1200, 1600, 1.0]] * 2, np.float32)
    rois = eng.rois_batch(ims, info)
    blob = (ims[0].astype(np.float32) - net_cpu.PIXEL_MEANS.astype(np.float64)).astype(np.float32)[None]
    ref = net_cpu.forward(blob, weights)
    assert ref["rpn_cls_score"].shape == (1, 75, 100, 20)
    want, _ = postproc.proposal_layer(ref["rpn_cls_prob_reshape"], ref["rpn_bbox_pred"], info[:1])
    got = rois[0]
    assert got.shape[0] == 1000 and want.shape[0] == 1000
    assert rows_matched(got, want) >= 0.995                  # all 1000 rows, not only the strongest


def test_config5_mixed_shapes_oriented_connector(weights):
    """BASELINE.json configs[4]: a mix of 600x900 and 900x600 images (two shape buckets) through the
    reference call sequence with DETECT_MODE 'O' (oriented text-line connector)."""
    from ctpn_b200 import Session
    from lib.fast_rcnn.config import cfg
    from lib.fast_rcnn.test import test_ctpn
    from lib.networks.factory import get_network
    from lib.text_connector.detectors import TextDetector
    from oracle import textline
    sess = Session(weights, planes=2)
    net = get_network("VGGnet_test")
    old = cfg.TEST.DETECT_MODE
    cfg.TEST.DETECT_MODE = "O"
    try:
        for seed, (h, w) in [(50, (600, 900)), (51, (900, 600)), (52, (600, 900))]:
            im = synth.make_image(seed, h, w)
            scores, boxes = test_ctpn(sess, net, im)
            assert boxes.shape[0] == scores.shape[0] > 0
            assert boxes[:, [0, 2]].max() <= w - 1 and boxes[:, [1, 3]].max() <= h - 1
            lines = TextDetector().detect(boxes, scores[:, np.newaxis], im.shape[:2])
            want = textline.detect(boxes, scores[:, np.newaxis], im.shape[:2], mode="O")   # same proposals -> same lines
            np.testing.assert_array_equal(lines, want)
    finally:
        cfg.TEST.DETECT_MODE = old


@pytest.mark.parametrize("h,w", [(50, 70), (16, 16), (33, 129)])
def test_tiny_and_odd_image_sizes(weights, h, w):
    """Ragged sizes: feature maps of 3x4, 1x1 and 2x8 cells; every pool level floors an odd dimension."""
    from ctpn_b200 import Engine
    eng = Engine(weights, planes=3)
    im = synth.make_image(60 + h, h, w)
    cls, bbox = eng.forward_heads(torch.from_numpy(im[None]).cuda())
    blob = im.astype(np.float32)
    blob -= net_cpu.PIXEL_MEANS
    ref = net_cpu.forward(blob[None], weights, dtype=torch.float64)
    assert tuple(cls.shape) == ref["rpn_cls_score"].shape
    assert np.abs(cls.cpu().numpy() - ref["rpn_cls_score"]).max() < 1e-3
    assert np.abs(bbox.cpu().numpy() - ref["rpn_bbox_pred"]).max() < 1e-3


def test_errors_are_reported(weights):
    from ctpn_b200 import CtpnError, Engine, _native as N
    eng = Engine(None)
    with pytest.raises(CtpnError, match="has not been set"):
        eng.forward_heads(torch.zeros((1, 64, 64, 3), dtype=torch.uint8, device="cuda"))
    with pytest.raises(CtpnError):
        eng.forward_heads(torch.zeros((1, 8, 64, 3), dtype=torch.uint8, device="cuda"))      # smaller than one cell
    assert N.lib.ctpn_device_ok(99) != 0 and "device" in N.last_error()


def test_detect_list_buckets_mixed_shapes(weights):
    from ctpn_b200 import Engine
    eng = Engine(weights, planes=2)
    shapes = [(64, 96), (96, 64), (64, 96), (48, 80), (96, 64)]
    ims = [synth.make_image(70 + i, h, w) for i, (h, w) in enumerate(shapes)]
    res = eng.detect_list(ims, max_batch=2)
    assert len(res) == len(ims)
    for im, (s, b) in zip(ims, res):
        s1, b1 = eng.detect(im)
        np.testing.assert_array_equal(s, s1)
        np.testing.assert_array_equal(b, b1)
