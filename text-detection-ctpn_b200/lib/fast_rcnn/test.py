"""test_ctpn(sess, net, im) -> (scores, boxes): the inference entry point of
lib/fast_rcnn/test.py:40-58, same signature and results, running on the H100 engine.

Host pre-processing follows test.py:7-31 (float32 copy, mean subtraction, rescale to
TEST.SCALES / TEST.MAX_SIZE with cv2.INTER_LINEAR).  When no rescale is needed and the image is
uint8, the uint8 pixels are fed directly: the engine's conv1_1 applies the identical
float32(double(v) - mean) subtraction on the device, so the result is bitwise the same blob."""
import cv2
import numpy as np

from .config import cfg
from lib.utils.blob import im_list_to_blob


def _im_scale(im_shape):
    im_size_min = np.min(im_shape[0:2])
    im_size_max = np.max(im_shape[0:2])
    scales = []
    for target_size in cfg.TEST.SCALES:
        im_scale = float(target_size) / float(im_size_min)
        if np.round(im_scale * im_size_max) > cfg.TEST.MAX_SIZE:
            im_scale = float(cfg.TEST.MAX_SIZE) / float(im_size_max)
        scales.append(im_scale)
    return scales


def _get_image_blob(im):
    scales = _im_scale(im.shape)
    if im.dtype == np.uint8 and len(scales) == 1 and scales[0] == 1.0:
        return im[None], np.array(scales)          # mean subtraction is fused into conv1_1
    im_orig = im.astype(np.float32, copy=True)
    im_orig -= cfg.PIXEL_MEANS
    processed = [cv2.resize(im_orig, None, None, fx=s, fy=s, interpolation=cv2.INTER_LINEAR) for s in scales]
    return im_list_to_blob(processed), np.array(scales)


def _get_blobs(im, rois):
    blobs = {'data': None, 'rois': None}
    blobs['data'], im_scale_factors = _get_image_blob(im)
    return blobs, im_scale_factors


def test_ctpn(sess, net, im, boxes=None):
    blobs, im_scales = _get_blobs(im, boxes)
    if cfg.TEST.HAS_RPN:
        im_blob = blobs['data']
        blobs['im_info'] = np.array([[im_blob.shape[1], im_blob.shape[2], im_scales[0]]], dtype=np.float32)
        feed_dict = {net.data: blobs['data'], net.im_info: blobs['im_info'], net.keep_prob: 1.0}
    else:
        raise NotImplementedError("only the RPN test path (cfg.TEST.HAS_RPN) exists in CTPN")
    rois = sess.run([net.get_output('rois')[0]], feed_dict=feed_dict)
    rois = rois[0]
    scores = rois[:, 0]
    assert len(im_scales) == 1, "Only single-image batch implemented"
    boxes = rois[:, 1:5] / im_scales[0]
    return scores, boxes
