"""Frozen-graph demo with the call structure of the reference's ctpn/demo_pb.py:55-98: weights from data/ctpn.pb
(ctpn/generate_pb.py:36-40 wrote it; read here without TensorFlow by ctpn_b200.tf_import), head tensors fetched by their
graph names, proposal_layer called DIRECTLY by the script (demo_pb.py:92) -- the one place in the reference where the
operator interface of lib/rpn_msr/proposal_layer_tf.py is used without tf.py_func -- then TextDetector and draw_boxes.

    python ctpn/demo_pb.py [--pb data/ctpn.pb] [--images 'data/demo/*'] [--planes 2]
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

from lib.fast_rcnn.config import cfg, cfg_from_file                     # noqa: E402
from lib.fast_rcnn.test import _get_blobs                                # noqa: E402
from lib.text_connector.detectors import TextDetector                   # noqa: E402
from lib.text_connector.text_connect_cfg import Config as TextLineCfg    # noqa: E402
from lib.rpn_msr.proposal_layer_tf import proposal_layer                 # noqa: E402
from ctpn.demo import RESULTS_DIR, draw_boxes, resize_im                 # noqa: E402,F401  (same helpers as demo.py)


def detect_pb(sess, im_name):
    """One image through the frozen-graph path (the loop body of demo_pb.py:82-98); returns the text lines."""
    input_img = sess.graph.get_tensor_by_name('Placeholder:0')
    output_cls_prob = sess.graph.get_tensor_by_name('Reshape_2:0')
    output_box_pred = sess.graph.get_tensor_by_name('rpn_bbox_pred/Reshape_1:0')
    img = cv2.imread(im_name)
    img, scale = resize_im(img, scale=TextLineCfg.SCALE, max_scale=TextLineCfg.MAX_SCALE)
    blobs, im_scales = _get_blobs(img, None)
    if cfg.TEST.HAS_RPN:
        im_blob = blobs['data']
        blobs['im_info'] = np.array([[im_blob.shape[1], im_blob.shape[2], im_scales[0]]], dtype=np.float32)
    cls_prob, box_pred = sess.run([output_cls_prob, output_box_pred], feed_dict={input_img: blobs['data']})
    rois, _ = proposal_layer(cls_prob, box_pred, blobs['im_info'], 'TEST', anchor_scales=cfg.ANCHOR_SCALES)
    scores = rois[:, 0]
    boxes = rois[:, 1:5] / im_scales[0]
    boxes = TextDetector().detect(boxes, scores[:, np.newaxis], img.shape[:2])
    draw_boxes(img, im_name, boxes, scale)
    return boxes


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--pb", default="data/ctpn.pb")
    ap.add_argument("--planes", type=int, default=2,
                    help="conv arithmetic: 1-3 bf16 planes, 4 = F16F8 (2 tensor-core units per MAC), 5 = bf16x3 with promoted accumulation")
    ap.add_argument("--images", default=None)
    ap.add_argument("--cfg", default=os.path.join(_PKG, 'ctpn', 'text.yml'))
    args = ap.parse_args(argv)
    if os.path.exists(RESULTS_DIR):
        shutil.rmtree(RESULTS_DIR)
    os.makedirs(RESULTS_DIR)
    cfg_from_file(args.cfg)
    from ctpn_b200 import Session
    sess = Session(planes=args.planes, device=cfg.GPU_ID)
    try:
        sess.restore(args.pb)                      # tf.import_graph_def of the frozen GraphDef (demo_pb.py:66-70)
    except (OSError, KeyError, ValueError) as e:
        raise SystemExit('Check your frozen graph {:s}: {}'.format(args.pb, e))
    pattern = args.images
    im_names = sorted(glob.glob(pattern)) if pattern else (glob.glob(os.path.join(cfg.DATA_DIR, 'demo', '*.png')) +
                                                            glob.glob(os.path.join(cfg.DATA_DIR, 'demo', '*.jpg')))
    for im_name in im_names:
        print('~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~~')
        print(('Demo for {:s}'.format(im_name)))
        detect_pb(sess, im_name)


if __name__ == '__main__':
    main()
