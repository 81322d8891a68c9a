"""GPU: ragged batches -- images of different sizes on one canvas (ctpn_net_forward_ragged, ctpn_proposals_ragged,
Engine.detect_ragged).  The contract is per image and bit for bit: the heads inside each image's feature extent and its
rois / index / count equal a run of that image alone, in every arithmetic, whatever the canvas holds outside the image."""
import numpy as np
import pytest
import torch

from oracle import net_cpu, synth

pytestmark = pytest.mark.gpu

# canvas 80 x 224.  63 is odd at every pool level (63 31 15 7 3), as is 159 (159 79 39 19 9); 203 and 129 are odd at
# full resolution; 16 x 16 is the smallest image; 80 x 224 fills the canvas; 80 x 159 is narrower and 47 x 224 shorter.
SIZES = [(63, 203), (33, 129), (16, 16), (80, 224), (80, 159), (47, 224)]
MODES = ["bf16", "bf16x2", "bf16x3", "bf16x3p", "f16f8"]
CONV_TAPS = [("conv1_1", 0, 64), ("conv1_2+pool", 1, 64), ("conv2_1", 1, 128), ("conv2_2+pool", 2, 128), ("conv3_1", 2, 256),
             ("conv3_2", 2, 256), ("conv3_3+pool", 3, 256), ("conv4_1", 3, 512), ("conv4_2", 3, 512), ("conv4_3+pool", 4, 512),
             ("conv5_1", 4, 512), ("conv5_2", 4, 512), ("conv5_3", 4, 512), ("rpn_conv/3x3", 4, 512), ("lstm_out", 4, 256)]


@pytest.fixture(scope="module")
def weights():
    return synth.make_weights(0)


def canvas_of(images, fill="zero", seed=0):
    """[B, H, W, 3] canvas of the images (uint8 or float32); padding zero, random bytes or NaN."""
    H = max(im.shape[0] for im in images)
    W = max(im.shape[1] for im in images)
    dt = images[0].dtype
    rs = np.random.RandomState(seed)
    if fill == "zero":
        c = np.zeros((len(images), H, W, 3), dt)
    elif fill == "random":
        c = rs.randint(0, 256, size=(len(images), H, W, 3)).astype(dt)
    else:
        c = np.full((len(images), H, W, 3), np.nan, dt)
    for b, im in enumerate(images):
        c[b, :im.shape[0], :im.shape[1]] = im
    return c


def make_images(sizes, seed0=20):
    return [synth.make_image(seed0 + i, h, w) for i, (h, w) in enumerate(sizes)]


def ragged_run(eng, canvas, sizes):
    """heads + proposals of a ragged batch: (cls, bbox, rois, index, count) as CUDA tensors."""
    B = len(sizes)
    dev = torch.from_numpy(canvas).cuda()
    cls, bbox = eng.forward_heads(dev, sizes=sizes)
    info = torch.tensor([[h, w, 1.0] for h, w in sizes], dtype=torch.float32)
    feat = [(h >> 4, w >> 4) for h, w in sizes]
    rois, index, count = eng.proposals(cls, bbox, info, feat_sizes=feat)
    assert rois.shape[0] == B
    return cls, bbox, rois, index, count


def single_run(eng, im):
    h, w = im.shape[:2]
    cls, bbox = eng.forward_heads(torch.from_numpy(np.ascontiguousarray(im[None])).cuda())
    rois, index, count = eng.proposals(cls, bbox, torch.tensor([[h, w, 1.0]], dtype=torch.float32))
    return cls, bbox, rois, index, count


def assert_image_equal(ragged, single, b, size, what=""):
    cls, bbox, rois, index, count = ragged
    scls, sbbox, srois, sindex, scount = single
    fh, fw = size[0] >> 4, size[1] >> 4
    assert torch.equal(cls[b, :fh, :fw], scls[0]), "%s image %d %s: cls heads differ" % (what, b, size)
    assert torch.equal(bbox[b, :fh, :fw], sbbox[0]), "%s image %d %s: bbox heads differ" % (what, b, size)
    assert int(count[b]) == int(scount[0]), "%s image %d %s: count %d vs %d" % (what, b, size, int(count[b]), int(scount[0]))
    n = int(scount[0])
    assert torch.equal(rois[b, :n], srois[0, :n]), "%s image %d %s: rois differ" % (what, b, size)
    assert torch.equal(index[b, :n], sindex[0, :n]), "%s image %d %s: index differs" % (what, b, size)


@pytest.mark.parametrize("mode", MODES)
def test_each_mode_equals_single_image_runs(weights, mode):
    from ctpn_b200 import Engine
    images = make_images(SIZES)
    eng = Engine(weights, mode=mode)
    ragged = ragged_run(eng, canvas_of(images, "random"), SIZES)     # f16f8: the ragged batch calibrates the scales
    for b, im in enumerate(images):
        assert_image_equal(ragged, single_run(eng, im), b, SIZES[b], mode)


def test_padding_content_is_ignored(weights):
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="bf16x2")
    images = make_images(SIZES)
    base = ragged_run(eng, canvas_of(images, "zero"), SIZES)
    noisy = ragged_run(eng, canvas_of(images, "random", seed=3), SIZES)
    blobs = [(im.astype(np.float32) - net_cpu.PIXEL_MEANS).astype(np.float32) for im in images]
    fbase = ragged_run(eng, canvas_of(blobs, "zero"), SIZES)
    fnan = ragged_run(eng, canvas_of(blobs, "nan"), SIZES)
    for b, (h, w) in enumerate(SIZES):
        fh, fw = h >> 4, w >> 4
        for x, y in ((base, noisy), (fbase, fnan)):
            assert torch.equal(x[0][b, :fh, :fw], y[0][b, :fh, :fw]) and torch.equal(x[1][b, :fh, :fw], y[1][b, :fh, :fw])
            assert torch.equal(x[2][b], y[2][b]) and torch.equal(x[3][b], y[3][b]) and int(x[4][b]) == int(y[4][b])
        assert torch.isfinite(fnan[0][b, :fh, :fw]).all()


@pytest.mark.parametrize("mode", ["bf16x2", "bf16x3p", "f16f8"])
def test_every_tap_is_zero_outside_the_extents(weights, mode):
    from ctpn_b200 import Engine
    images = make_images(SIZES)
    canvas = canvas_of(images, "random", seed=5)
    B, H, W, _ = canvas.shape
    eng = Engine(weights, mode=mode, keep_activations=True)
    eng.forward_heads(torch.from_numpy(canvas).cuda(), sizes=SIZES)
    torch.cuda.synchronize()
    for name, k, ch in CONV_TAPS:
        t = eng.tap(name).cpu().numpy().reshape(B, H >> k, W >> k, ch)
        for b, (h, w) in enumerate(SIZES):
            eh, ew = h >> k, w >> k
            outside = np.concatenate([t[b, eh:].ravel(), t[b, :eh, ew:].ravel()])
            assert not outside.any(), "%s %s image %d: %d nonzero values outside %dx%d" % (mode, name, b, np.count_nonzero(outside), eh, ew)
            assert t[b, :eh, :ew].any(), "%s %s image %d: all zero inside" % (mode, name, b)


def test_proposals_ignore_padded_cells(weights):
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="bf16x2")
    images = make_images(SIZES)
    cls, bbox, _, _, _ = ragged_run(eng, canvas_of(images), SIZES)
    cls, bbox = cls.clone(), bbox.clone()
    feat = [(h >> 4, w >> 4) for h, w in SIZES]
    for b, (fh, fw) in enumerate(feat):
        for t in (cls, bbox):
            t[b, fh:] = float("nan")
            t[b, :, fw:] = float("nan")
    info = torch.tensor([[h, w, 1.0] for h, w in SIZES], dtype=torch.float32)
    for logit in (True, False):
        c = cls if logit else torch.sigmoid(cls)      # any finite probabilities inside, NaN outside
        rois, index, count = eng.proposals(c, bbox, info, cls_is_logit=logit, feat_sizes=feat)
        for b, (fh, fw) in enumerate(feat):
            s_rois, s_index, s_count = eng.proposals(c[b:b + 1, :fh, :fw].contiguous(), bbox[b:b + 1, :fh, :fw].contiguous(),
                                                     info[b:b + 1], cls_is_logit=logit)
            n = int(s_count[0])
            assert int(count[b]) == n and n > 0
            assert torch.equal(rois[b, :n], s_rois[0, :n]) and torch.equal(index[b, :n], s_index[0, :n])
            assert int(index[b, :n].max()) < fh * fw * 10


@pytest.mark.parametrize("mode", ["f16f8", "bf16x2"])
def test_realistic_batch_of_32(weights, mode):
    """Blob sizes the demo produces (600 x 600..1000, or < 600 x 1000 beyond 5:3): the 1/16 maps are row-stacked, the big
    layers run one CTA per SM and the BiLSTM at 40 rows per cluster."""
    from ctpn_b200 import Engine
    rs = np.random.RandomState(5)
    sizes = [(600, int(rs.randint(600, 1001))) if i % 4 != 3 else (int(rs.randint(360, 600)), 1000) for i in range(32)]
    sizes[31] = (600, 1000)
    images = make_images(sizes, seed0=100)
    eng = Engine(weights, mode=mode)
    ragged = ragged_run(eng, canvas_of(images, "random"), sizes)
    for b in (0, 15, 31):
        assert_image_equal(ragged, single_run(eng, images[b]), b, sizes[b], mode)


def test_ragged_bf16x3p_against_float64(weights):
    from ctpn_b200 import Engine
    sizes = [(96, 160), (63, 203), (33, 129)]
    images = make_images(sizes, seed0=7)
    cls, bbox, _, _, _ = ragged_run(Engine(weights, mode="bf16x3p"), canvas_of(images, "random"), sizes)
    for b, (im, (h, w)) in enumerate(zip(images, sizes)):
        blob = (im.astype(np.float32) - net_cpu.PIXEL_MEANS.astype(np.float64)).astype(np.float32)[None]
        ref = net_cpu.forward(blob, weights, dtype=torch.float64)
        fh, fw = h >> 4, w >> 4
        d_cls = float(np.abs(cls[b, :fh, :fw].cpu().numpy() - ref["rpn_cls_score"][0]).max())
        d_box = float(np.abs(bbox[b, :fh, :fw].cpu().numpy() - ref["rpn_bbox_pred"][0]).max())
        assert d_cls < 3e-5 and d_box < 1e-5, (b, d_cls, d_box)    # the bounds of test_promote_gpu's 600x900 check


def test_detect_ragged_end_to_end(weights):
    from ctpn_b200 import Engine
    eng = Engine(weights, mode="bf16x2")
    sizes = [(96, 160), (160, 96), (63, 203), (129, 33), (80, 80), (112, 208), (200, 64)]
    ims = make_images(sizes, seed0=40)
    images, scales = [], []
    for i, im in enumerate(ims):
        if i % 2:
            images.append((im.astype(np.float32) - net_cpu.PIXEL_MEANS).astype(np.float32))
            scales.append(0.75)
        else:
            images.append(im)
            scales.append(1.0)
    got = eng.detect_ragged(images, im_scales=scales, max_batch=2)
    assert len(got) == len(images)
    for im, s, (scores, boxes) in zip(images, scales, got):
        want_s, want_b = eng.detect(im, im_scale=s)
        assert np.array_equal(scores, want_s) and np.array_equal(boxes, want_b)
    with pytest.raises(ValueError):
        eng.detect_ragged([ims[0][:15]])
    with pytest.raises(ValueError):
        eng.detect_ragged(ims[:2], im_scales=[1.0])
    with pytest.raises(ValueError):
        eng.forward_heads(torch.zeros((1, 32, 32, 3), dtype=torch.uint8, device="cuda"), sizes=[(33, 32)])


def test_demo_batch_writes_the_same_results(weights, tmp_path, monkeypatch):
    """ctpn/demo.py --batch 4 == --batch 1 (bf16x2; F16F8 would calibrate on a different first batch).  One image is wider
    than 5:3, so its blob needs _get_image_blob's float rescale to MAX_SIZE."""
    cv2 = pytest.importorskip("cv2")
    from ctpn import demo
    npz = str(tmp_path / "w.npz")
    np.savez(npz, **weights)
    folder = tmp_path / "images"
    folder.mkdir()
    for i, (h, w) in enumerate([(300, 400), (480, 360), (200, 500), (240, 240), (350, 420)]):
        cv2.imwrite(str(folder / ("im_%d.png" % i)), synth.make_image(60 + i, h, w))
    out = {}
    for batch in (1, 4):
        res = tmp_path / ("results_%d" % batch)
        monkeypatch.setattr(demo, "RESULTS_DIR", str(res))
        demo.main(["--weights", npz, "--planes", "2", "--images", str(folder / "*.png"), "--batch", str(batch)])
        out[batch] = {p.name: p.read_bytes() for p in sorted(res.glob("res_*.txt"))}
    assert len(out[1]) == 5 and out[1] == out[4]
