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
the output files are the same.  --gpu-decode (with --device-frontend) decodes the JPEG files on the GPU
(torchvision.io.decode_jpeg, nvJPEG) and passes the RGB tensors to the same calls, which read them in place: only the
compressed files cross the bus.  nvJPEG's pixels are not cv2.imread's (another IDCT and chroma upsampling), so the files
written equal those of --device-frontend on the decoded pixels, not on cv2's.  Files nvJPEG cannot stand in for -- not
JPEG, an EXIF orientation other than 1 (cv2.imread rotates those), or a frame other than baseline or progressive
Huffman with 1 or 3 components -- are read with cv2.imread and uploaded instead.
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
GPU_DECODE = False            # --gpu-decode: JPEG files decoded on the GPU (nvJPEG through torchvision), read in place


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


def jpeg_on_gpu(data):
    """Whether nvJPEG's decode of the file `data` (bytes) stands in for cv2.imread's, judged from its markers alone: a JPEG
    whose frame is baseline (SOF0) or progressive (SOF2) Huffman with 1 or 3 components, and whose EXIF orientation, if it
    has one, is 1 (cv2.imread rotates the others; the CUDA decode does not)."""
    if data[:2] != b"\xff\xd8":
        return False
    i, frame = 2, None
    while i + 4 <= len(data) and frame is None:
        if data[i] != 0xFF:
            return False
        marker = data[i + 1]
        if marker == 0xFF:                     # fill byte
            i += 1
            continue
        n = int.from_bytes(data[i + 2:i + 4], "big")
        seg = data[i + 4:i + 2 + n]
        if marker == 0xE1 and seg[:6] == b"Exif\x00\x00" and exif_orientation(seg[6:]) not in (None, 1):
            return False
        if 0xC0 <= marker <= 0xCF and marker not in (0xC4, 0xC8, 0xCC):     # SOFn (C4 DHT, C8 JPG, CC DAC are not frames)
            frame = (marker, seg[5] if len(seg) > 5 else 0)
        if marker == 0xDA:                     # scan before any frame
            return False
        i += 2 + n
    return frame is not None and frame[0] in (0xC0, 0xC2) and frame[1] in (1, 3)


def exif_orientation(tiff):
    """The Orientation tag (0x0112) of IFD0 of an EXIF TIFF block, or None."""
    if len(tiff) < 8 or tiff[:2] not in (b"II", b"MM"):
        return None
    order = "little" if tiff[:2] == b"II" else "big"
    ifd = int.from_bytes(tiff[4:8], order)
    if ifd + 2 > len(tiff):
        return None
    for k in range(int.from_bytes(tiff[ifd:ifd + 2], order)):
        e = tiff[ifd + 2 + 12 * k:ifd + 14 + 12 * k]
        if len(e) == 12 and int.from_bytes(e[:2], order) == 0x0112:
            return int.from_bytes(e[8:10], order)
    return None


def read_on_device(names):
    """The files as CUDA uint8 [H, W, 3] RGB tensors: JPEGs nvJPEG can stand in for decoded on the GPU in one batched call
    (ImageReadMode.RGB: cv2.imread makes three channels of a grayscale JPEG too), every other file read by cv2.imread,
    flipped to RGB on the host and uploaded, so that the engine's call takes device tensors only."""
    import torch
    from torchvision.io import ImageReadMode, decode_jpeg
    datas = []
    for name in names:
        with open(name, "rb") as f:
            datas.append(f.read())
    gpu = [i for i, d in enumerate(datas) if jpeg_on_gpu(d)]
    out = [None] * len(names)
    if gpu:
        decoded = decode_jpeg([torch.frombuffer(bytearray(datas[i]), dtype=torch.uint8) for i in gpu], mode=ImageReadMode.RGB,
                              device="cuda")
        for i, t in zip(gpu, decoded):
            out[i] = t.permute(1, 2, 0)
    for i, name in enumerate(names):
        if out[i] is None:
            out[i] = torch.from_numpy(np.ascontiguousarray(cv2.imread(name)[:, :, ::-1])).cuda()
    return out


def read_images(names):
    """The images of a batch and their channel order: cv2.imread's BGR arrays, or with --gpu-decode RGB device tensors."""
    if GPU_DECODE:
        return read_on_device(names), "RGB"
    return [cv2.imread(name) for name in names], "BGR"


def ctpn_batch_device(sess, image_names):
    """ctpn_batch with resize_im and _get_image_blob on the device (Engine.rois_images): the images go up as read (or are
    decoded on the device with --gpu-decode), and the resized images come back for draw_boxes.  Same TextDetector,
    draw_boxes and output files per image."""
    timer = Timer()
    timer.tic()
    imgs, channels = read_images(image_names)
    if DEVICE_LINES:        # the lines of TextDetector(native=True), built on the device; only they come back with the images
        res = sess.engine.detect_lines_images(imgs, mode=cfg.TEST.DETECT_MODE, return_resized=True, scale=TextLineCfg.SCALE,
                                              max_scale=TextLineCfg.MAX_SCALE, cfg=native_cfg(), channels=channels)
        for name, (boxes, scale, img) in zip(image_names, res):
            draw_boxes(img, name, boxes, scale)
            print('{:s}: {:d} text lines'.format(name, boxes.shape[0]))
        timer.toc()
        print(('Detection of {:d} images took {:.3f}s').format(len(image_names), timer.total_time))
        return
    res = sess.engine.rois_images(imgs, return_resized=True, scale=TextLineCfg.SCALE, max_scale=TextLineCfg.MAX_SCALE,
                                  channels=channels)
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
    decoded = (read_images([name])[0][0] for name in image_names)
    kw = dict(max_batch=batch, return_resized=True, scale=TextLineCfg.SCALE, max_scale=TextLineCfg.MAX_SCALE,
              channels="RGB" if GPU_DECODE else "BGR")
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
    ap.add_argument("--gpu-decode", action="store_true",
                    help="with --device-frontend: decode JPEG files on the GPU (torchvision nvJPEG; lazily, one file at a time, "
                         "with --stream) and read them in place.  nvJPEG's pixels differ from cv2.imread's, so the files equal "
                         "those of --device-frontend on the decoded pixels, not on cv2's.  Other files, and JPEGs with an EXIF "
                         "rotation or an unusual frame, are read with cv2 and uploaded")
    args = ap.parse_args(argv)
    if args.stream and not args.device_frontend:
        ap.error("--stream needs --device-frontend (and --batch N with N > 1)")
    if args.device_frontend and args.batch <= 1:
        ap.error("--device-frontend needs --batch N with N > 1")
    if args.device_lines and not args.device_frontend:
        ap.error("--device-lines needs --device-frontend (and --batch N with N > 1)")
    if args.gpu_decode and not args.device_frontend:
        ap.error("--gpu-decode needs --device-frontend (and --batch N with N > 1)")
    global NATIVE_CONNECTOR, DEVICE_LINES, GPU_DECODE
    NATIVE_CONNECTOR = args.native_connector
    DEVICE_LINES = args.device_lines
    GPU_DECODE = args.gpu_decode
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
