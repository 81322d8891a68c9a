"""Command-line demo with the call structure of the reference's ctpn/demo.py:

    python ctpn/demo.py [--weights CKPT_DIR|model.ckpt|ctpn.pb|W.npz] [--planes 2] [--images 'data/demo/*']

ctpn(sess, net, image_name) keeps the reference signature (demo.py:55-68): read image, resize
(short side 600, long side <= 1200), test_ctpn, TextDetector, write data/results/res_<stem>.txt
and the annotated image.  `sess` is a ctpn_b200.Session (replaces tf.Session + Saver.restore).
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
from lib.fast_rcnn.test import test_ctpn                 # noqa: E402
from lib.utils.timer import Timer                        # noqa: E402
from lib.text_connector.detectors import TextDetector   # noqa: E402
from lib.text_connector.text_connect_cfg import Config as TextLineCfg  # noqa: E402

RESULTS_DIR = "data/results"
NATIVE_CONNECTOR = False      # --native-connector: C++ text-line connector of the library instead of the Python one


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
    args = ap.parse_args(argv)
    global NATIVE_CONNECTOR
    NATIVE_CONNECTOR = args.native_connector
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
    for im_name in sorted(glob.glob(args.images)):
        print('~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~')
        print('Demo for {:s}'.format(im_name))
        ctpn(sess, net, im_name)


if __name__ == '__main__':
    main()
