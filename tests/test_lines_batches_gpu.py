"""GPU: Engine.detect_lines_batches, the rois -> host connector pipeline behind bench.py's end-to-end text-line figure.  For
every image of every batch its lines must be, as float64 bits, text_lines(rois[:, 1:5] / np.float64(scale), rois[:, 0],
frame, mode) on rois_batch's rois of that batch -- what test_ctpn and TextDetector compute -- in modes H and O, on 1 and 8
connector threads, for successive batches of different shapes at scale 1 and for blobs made at scales other than 1, where
the frame is the image's size (im_hw) and not the blob's size divided by the scale."""
import numpy as np
import pytest

from oracle import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from ctpn_b200 import Engine
    return Engine(synth.make_weights(0), mode="bf16x2")


def lines_want(eng, batch, im_info, scale, frame, mode):
    from ctpn_b200.textlines import text_lines
    rois = eng.rois_batch(batch, None if im_info is None else np.asarray(im_info, np.float32))
    return [text_lines(r[:, 1:5] / np.float64(scale), r[:, 0], frame or batch.shape[1:3], mode) for r in rois]


def same_lines(got, want, what):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.dtype == w.dtype == np.float64 and g.shape == w.shape, (what, i, g.shape, w.shape)
        assert np.array_equal(g.view(np.uint64), w.view(np.uint64)), (what, i)


def test_successive_batches_of_different_shapes_at_scale_1(eng):
    shapes = [(3, 600, 900), (2, 900, 600), (4, 480, 640), (1, 600, 900), (3, 600, 900)]
    batches = [np.stack([synth.make_image(300 + 10 * k + i, h, w) for i in range(B)]) for k, (B, h, w) in enumerate(shapes)]
    for mode in ("H", "O"):
        want = [lines_want(eng, b, None, 1.0, None, mode) for b in batches]
        assert sum(len(l) for w in want for l in w) > 0
        for workers in (1, 8):
            got = list(eng.detect_lines_batches(iter(batches), mode=mode, workers=workers))
            assert len(got) == len(batches)
            for k, (g, w) in enumerate(zip(got, want)):
                same_lines(g, w, (mode, workers, k))


def blob_batches(eng, h, w, n_batches, B, seed):
    """Blobs as _get_image_blob makes them from h x w photos (float32, mean-subtracted, rescaled on the device), with the
    float64 im_scale of test.py's rule; returns (host float32 batches, im_scale, blob (H, W))."""
    target, max_size = 600.0, 1000.0
    im_scale = target / min(h, w)
    if np.round(im_scale * max(h, w)) > max_size:
        im_scale = max_size / max(h, w)
    batches = []
    for k in range(n_batches):
        photos = np.stack([synth.make_image(seed + B * k + i, h, w) for i in range(B)])
        batches.append(eng.image_blob(photos, im_scale).cpu().numpy())
    return batches, im_scale, batches[0].shape[1:3]


# (h, w) of the photos: scale 1.6, 1000 / 1100 and 1000 / 1023 (blob width / scale rounds to 599 and 601, not 600), 600 / 1080
SCALED = [(375, 500), (1100, 600), (1023, 600), (1080, 1440)]


@pytest.mark.parametrize("h,w", SCALED, ids=["%dx%d" % s for s in SCALED])
def test_scaled_blobs_give_the_lines_of_test_ctpn(eng, h, w):
    batches, im_scale, (bh, bw) = blob_batches(eng, h, w, 3, 2, 400 + h)
    assert im_scale != 1.0
    wrong_frame = (int(round(bh / float(np.float32(im_scale)))), int(round(bw / float(np.float32(im_scale)))))
    print("%dx%d: scale %r, blob %dx%d, blob / float32 scale rounds to %s" % (h, w, im_scale, bh, bw, wrong_frame))
    if (h, w) in ((1100, 600), (1023, 600)):
        assert wrong_frame != (h, w)
    info = np.array([[bh, bw, im_scale]] * 2, np.float64)
    for mode in ("H", "O"):
        want = [lines_want(eng, b, info, im_scale, (h, w), mode) for b in batches]
        assert sum(len(l) for wl in want for l in wl) > 0
        for workers in (1, 8):
            got = list(eng.detect_lines_batches(iter(batches), mode=mode, im_info=info, workers=workers, im_hw=(h, w)))
            assert len(got) == len(batches)
            for k, (g, wl) in enumerate(zip(got, want)):
                same_lines(g, wl, (mode, workers, k))


def test_a_scale_other_than_1_needs_the_frame(eng):
    batches, im_scale, (bh, bw) = blob_batches(eng, 375, 500, 1, 1, 450)
    info = np.array([[bh, bw, im_scale]], np.float64)
    with pytest.raises(ValueError, match="im_hw"):
        next(eng.detect_lines_batches(iter(batches), im_info=info))
    with pytest.raises(ValueError, match="im_hw"):
        next(eng.detect_lines_batches(iter(batches), im_info=info, im_hw=(375, 500, 3)))
