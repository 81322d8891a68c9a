"""Command-line demo with the call structure of the reference's ctpn/demo.py:

    python ctpn/demo.py [--weights CKPT_DIR|model.ckpt|ctpn.pb|W.npz] [--planes 2] [--images 'data/demo/*'] [--batch N]

ctpn(sess, net, image_name) keeps the reference signature (demo.py:55-68): read image, resize
(short side 600, long side <= 1200), test_ctpn, TextDetector, write data/results/res_<stem>.txt
and the annotated image.  `sess` is a ctpn_b200.Session (replaces tf.Session + Saver.restore).
--batch N > 1 runs N images at a time through Engine.rois_ragged (images of different sizes in one batch), with the same
resize, blob, TextDetector and output files per image (ctpn_batch).  --device-frontend (with --batch N) runs the resize
and the blob on the GPU as well (Engine.rois_images, ctpn_batch_device); the output files are the same.
--device-lines (with --device-frontend) builds the text lines on the GPU too (Engine.detect_lines_images): the files equal
those of --device-frontend --native-connector.  --stream (with --device-frontend) reads and decodes the files one at a
time while earlier ones are uploaded and computed (Engine.stream_rois_images / stream_lines_images, ctpn_stream_device);
the output files are the same.
"""
from __future__ import print_function

import argparse
import glob
import os
import shutil
import sys

import cv2
import numpy as np

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)
sys.path.append(os.getcwd())

from lib.networks.factory import get_network            # noqa: E402
from lib.fast_rcnn.config import cfg, cfg_from_file     # noqa: E402
from lib.fast_rcnn.test import _get_image_blob, test_ctpn  # noqa: E402
from lib.utils.timer import Timer                        # noqa: E402
from lib.text_connector.detectors import TextDetector   # noqa: E402
from lib.text_connector.text_connect_cfg import Config as TextLineCfg, native_cfg  # noqa: E402

RESULTS_DIR = "data/results"
NATIVE_CONNECTOR = False      # --native-connector: C++ text-line connector of the library instead of the Python one
DEVICE_LINES = False          # --device-lines: the library's device connector on each batch's rois (Engine.detect_lines_images)


def resize_im(im, scale, max_scale=None):
    f = float(scale) / min(im.shape[0], im.shape[1])
    if max_scale is not None and f * max(im.shape[0], im.shape[1]) > max_scale:
        f = float(max_scale) / max(im.shape[0], im.shape[1])
    return cv2.resize(im, None, None, fx=f, fy=f, interpolation=cv2.INTER_LINEAR), f


def draw_boxes(img, image_name, boxes, scale):
    """Writes res_<stem>.txt ("min_x,min_y,max_x,max_y\\r\\n" in original-image pixels) and the
    annotated image (demo.py:28-52, including its scalar skip test on box[0..3])."""
    base_name = image_name.split('/')[-1]
    os.makedirs(RESULTS_DIR, exist_ok=True)
    with open(os.path.join(RESULTS_DIR, 'res_{}.txt'.format(base_name.split('.')[0])), 'w') as f:
        for box in boxes:
            if np.linalg.norm(box[0] - box[1]) < 5 or np.linalg.norm(box[3] - box[0]) < 5:
                continue
            color = (0, 255, 0) if box[8] >= 0.9 else (255, 0, 0)
            pts = [(int(box[0]), int(box[1])), (int(box[2]), int(box[3])), (int(box[6]), int(box[7])), (int(box[4]), int(box[5]))]
            for a, b in zip(pts, pts[1:] + pts[:1]):
                cv2.line(img, a, b, color, 2)
            xs = [int(box[i] / scale) for i in (0, 2, 4, 6)]
            ys = [int(box[i] / scale) for i in (1, 3, 5, 7)]
            f.write(','.join([str(min(xs)), str(min(ys)), str(max(xs)), str(max(ys))]) + '\r\n')
    img = cv2.resize(img, None, None, fx=1.0 / scale, fy=1.0 / scale, interpolation=cv2.INTER_LINEAR)
    cv2.imwrite(os.path.join(RESULTS_DIR, base_name), img)


def ctpn(sess, net, image_name):
    timer = Timer()
    timer.tic()
    img = cv2.imread(image_name)
    img, scale = resize_im(img, scale=TextLineCfg.SCALE, max_scale=TextLineCfg.MAX_SCALE)
    scores, boxes = test_ctpn(sess, net, img)
    textdetector = TextDetector(native=NATIVE_CONNECTOR)
    boxes = textdetector.detect(boxes, scores[:, np.newaxis], img.shape[:2])
    draw_boxes(img, image_name, boxes, scale)
    timer.toc()
    print(('Detection took {:.3f}s for {:d} object proposals').format(timer.total_time, boxes.shape[0]))


def ctpn_batch(sess, image_names):
    """ctpn() for several images at once: each is read, resized and turned into its blob as ctpn() / test_ctpn() do, the
    blobs run as ragged batches (Engine.rois_ragged), and each result goes through TextDetector and draw_boxes."""
    timer = Timer()
    timer.tic()
    imgs, scales, blobs, im_scales = [], [], [], []
    for name in image_names:
        img, scale = resize_im(cv2.imread(name), scale=TextLineCfg.SCALE, max_scale=TextLineCfg.MAX_SCALE)
        blob, im_scale = _get_image_blob(img)
        imgs.append(img)
        scales.append(scale)
        blobs.append(blob[0])
        im_scales.append(float(im_scale[0]))
    rois = sess.engine.rois_ragged(blobs, im_scales=im_scales)
    for name, img, scale, r, im_scale in zip(image_names, imgs, scales, rois, im_scales):
        scores, boxes = r[:, 0], r[:, 1:5] / np.float64(im_scale)      # the float64 division of test_ctpn
        textdetector = TextDetector(native=NATIVE_CONNECTOR)
        boxes = textdetector.detect(boxes, scores[:, np.newaxis], img.shape[:2])
        draw_boxes(img, name, boxes, scale)
        print('{:s}: {:d} text lines'.format(name, boxes.shape[0]))
    timer.toc()
    print(('Detection of {:d} images took {:.3f}s').format(len(image_names), timer.total_time))


def ctpn_batch_device(sess, image_names):
    """ctpn_batch with resize_im and _get_image_blob on the device (Engine.rois_images): the images go up as read, and
    the resized images come back for draw_boxes.  Same TextDetector, draw_boxes and output files per image."""
    timer = Timer()
    timer.tic()
    imgs = [cv2.imread(name) for name in image_names]
    if DEVICE_LINES:        # the lines of TextDetector(native=True), built on the device; only they come back with the images
        res = sess.engine.detect_lines_images(imgs, mode=cfg.TEST.DETECT_MODE, return_resized=True, scale=TextLineCfg.SCALE,
                                              max_scale=TextLineCfg.MAX_SCALE, cfg=native_cfg())
        for name, (boxes, scale, img) in zip(image_names, res):
            draw_boxes(img, name, boxes, scale)
            print('{:s}: {:d} text lines'.format(name, boxes.shape[0]))
        timer.toc()
        print(('Detection of {:d} images took {:.3f}s').format(len(image_names), timer.total_time))
        return
    res = sess.engine.rois_images(imgs, return_resized=True, scale=TextLineCfg.SCALE, max_scale=TextLineCfg.MAX_SCALE)
    for name, (r, im_scale, scale, img) in zip(image_names, res):
        scores, boxes = r[:, 0], r[:, 1:5] / np.float64(im_scale)      # the float64 division of test_ctpn
        textdetector = TextDetector(native=NATIVE_CONNECTOR)
        boxes = textdetector.detect(boxes, scores[:, np.newaxis], img.shape[:2])
        draw_boxes(img, name, boxes, scale)
        print('{:s}: {:d} text lines'.format(name, boxes.shape[0]))
    timer.toc()
    print(('Detection of {:d} images took {:.3f}s').format(len(image_names), timer.total_time))


def ctpn_stream_device(sess, image_names, batch):
    """ctpn_batch_device for the whole folder as one stream: every file is decoded when the pipeline asks for it
    (Engine.stream_rois_images / stream_lines_images pull a window of images at a time), and each image's files are
    written when its result arrives, while later images are still on their way."""
    timer = Timer()
    timer.tic()
    decoded = (cv2.imread(name) for name in image_names)
    kw = dict(max_batch=batch, return_resized=True, scale=TextLineCfg.SCALE, max_scale=TextLineCfg.MAX_SCALE)
    if DEVICE_LINES:
        results = sess.engine.stream_lines_images(decoded, mode=cfg.TEST.DETECT_MODE, cfg=native_cfg(), **kw)
    else:
        results = sess.engine.stream_rois_images(decoded, **kw)
    for name, res in zip(image_names, results):
        if DEVICE_LINES:
            boxes, scale, img = res
        else:
            r, im_scale, scale, img = res
            scores, boxes = r[:, 0], r[:, 1:5] / np.float64(im_scale)      # the float64 division of test_ctpn
            boxes = TextDetector(native=NATIVE_CONNECTOR).detect(boxes, scores[:, np.newaxis], img.shape[:2])
        draw_boxes(img, name, boxes, scale)
        print('{:s}: {:d} text lines'.format(name, boxes.shape[0]))
    timer.toc()
    print(('Detection of {:d} images took {:.3f}s').format(len(image_names), timer.total_time))


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--weights", default=None,
                    help="TF checkpoint prefix / directory, frozen .pb, VGG .npy or .npz (default: cfg.TEST.checkpoints_path, "
                         "like demo.py:88-90)")
    ap.add_argument("--planes", type=int, default=2, help="conv arithmetic: 1-3 bf16 planes, 4 = F16F8 (2 tensor-core units per MAC), 5 = bf16x3 with promoted accumulation")
    ap.add_argument("--images", default=os.path.join(cfg.DATA_DIR, 'demo', '*'))
    ap.add_argument("--cfg", default=os.path.join(_PKG, 'ctpn', 'text.yml'))
    ap.add_argument("--native-connector", action="store_true",
                    help="build the text lines with the library's C++ connector (same lines, float32-rounding agreement)")
    ap.add_argument("--batch", type=int, default=1,
                    help="images per ragged batch (Engine.detect_ragged); 1 = one image at a time through test_ctpn")
    ap.add_argument("--device-frontend", action="store_true",
                    help="with --batch N: run resize_im and the image blob on the GPU (Engine.rois_images) instead of cv2 on "
                         "the host; same output files")
    ap.add_argument("--device-lines", action="store_true",
                    help="with --device-frontend: build the text lines on the GPU as well (Engine.detect_lines_images); same "
                         "output files as --native-connector")
    ap.add_argument("--stream", action="store_true",
                    help="with --device-frontend: decode the files lazily and overlap decoding, upload and compute "
                         "(Engine.stream_rois_images / stream_lines_images); same output files")
    args = ap.parse_args(argv)
    if args.stream and not args.device_frontend:
        ap.error("--stream needs --device-frontend (and --batch N with N > 1)")
    if args.device_frontend and args.batch <= 1:
        ap.error("--device-frontend needs --batch N with N > 1")
    if args.device_lines and not args.device_frontend:
        ap.error("--device-lines needs --device-frontend (and --batch N with N > 1)")
    global NATIVE_CONNECTOR, DEVICE_LINES
    NATIVE_CONNECTOR = args.native_connector
    DEVICE_LINES = args.device_lines
    if os.path.exists(RESULTS_DIR):
        shutil.rmtree(RESULTS_DIR)
    os.makedirs(RESULTS_DIR)
    cfg_from_file(args.cfg)
    from ctpn_b200 import Session
    sess = Session(planes=args.planes, device=cfg.GPU_ID)
    net = get_network("VGGnet_test")
    print('Loading network VGGnet_test... ', end=' ')
    weights = args.weights if args.weights is not None else cfg.TEST.checkpoints_path
    try:        # demo.py:87-93: get_checkpoint_state(cfg.TEST.checkpoints_path) + saver.restore
        print('Restoring from {}...'.format(weights), end=' ')
        sess.restore(weights)
        print('done')
    except (OSError, KeyError, ValueError) as e:
        raise SystemExit('Check your pretrained {:s}: {}'.format(str(weights), e))
    im = 128 * np.ones((300, 300, 3), dtype=np.uint8)
    for _ in range(2):                                  # warm-up as demo.py:95-97
        test_ctpn(sess, net, im)
    if args.planes == 4:                                # F16F8: take the activation scales from the first real image, not from the flat
        sess.engine.recalibrate()                       # grey warm-up image
    names = sorted(glob.glob(args.images))
    if args.stream:
        print('~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~')
        ctpn_stream_device(sess, names, args.batch)
        return
    if args.batch > 1:
        for k in range(0, len(names), args.batch):
            print('~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~')
            (ctpn_batch_device if args.device_frontend else ctpn_batch)(sess, names[k:k + args.batch])
        return
    for im_name in names:
        print('~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~')
        print('Demo for {:s}'.format(im_name))
        ctpn(sess, net, im_name)


if __name__ == '__main__':
    main()
