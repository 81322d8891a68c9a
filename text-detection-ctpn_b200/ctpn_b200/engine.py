"""Engine: host-side driver of the H100 CTPN hot path.

PyTorch is used only as plumbing (device memory, streams, pinned buffers); all
compute is in libctpn_b200.so (see include/ctpn_b200.h).  One Engine == one GPU.

    eng = Engine(weights, planes=2)              # weights: {tf_variable_name: ndarray}
    scores, boxes = eng.detect(im)               # == lib.fast_rcnn.test.test_ctpn
    results = eng.detect_batch(uint8_batch)      # [B,H,W,3] -> list of (scores, boxes)
    results = eng.detect_ragged([im0, im1, ...])  # images of different sizes, batched on shared canvases
    results = eng.detect_images([photo0, ...])   # raw photos: resize_im + _get_image_blob on the device, then as above
    lines = eng.detect_lines_images([photo0, ...])  # ... and the text-line connector on the device: ctpn() per image
    for scores, boxes, f in eng.stream_images(cv2.imread(p) for p in paths): ...   # the same from any iterable, in input
                                                 # order, with packing, upload, compute and download overlapped

`planes` / `mode` select the arithmetic of the tensor-core layers (see include/ctpn_b200.h); accumulation is always
float32:  1 / "bf16" = bf16 operands (1 unit per MAC);  2 / "bf16x2" = bf16x2 split, ~16 mantissa bits (3 units);
3 / "bf16x3" = bf16x3 split, exact float32 operands (6 units), but the tensor core's truncating accumulation leaves the
head logits ~10x further from float64 than a float32 computation (DESIGN.md section 5);  5 / "bf16x3p" = bf16x3 with the
main accumulator promoted to round-to-nearest float32 every 64 channels of a tap (CTPN_F_PROMOTE; 6 units);
4 / "f16f8" = fp16 operands + e4m3 cross terms for the 3x3 layers (2 units; head logits within 1e-3 of float32, 6-8e-4
measured; activation scales calibrated on the first batch).
"""
import collections
import ctypes as C
import functools

import os

import numpy as np
import torch

from . import _native as N

# lib/fast_rcnn/config.py:147-183 defaults used by the test path
DEFAULT_CFG = dict(RPN_PRE_NMS_TOP_N=12000, RPN_POST_NMS_TOP_N=1000, RPN_NMS_THRESH=0.7, RPN_MIN_SIZE=8,
                   SCALES=(600,), MAX_SIZE=1000, FEAT_STRIDE=16, ANCHORS_PY2=False)


class Engine:
    MODES = {"bf16": 1, "bf16x2": 2, "bf16x3": 3, "f16f8": 4, "bf16x3p": 5}

    def __init__(self, weights=None, planes=2, device=0, cfg=None, conv_simt=False, keep_activations=False, streams=1, mode=None,
                 graph_max_batch=4):
        """graph_max_batch: batches of up to this many images run as a replayed CUDA graph per (shape, dtype) bucket (the ~25
        kernel launches of a step cost more than the kernels themselves at batch 1); 0 disables graphs.
        streams: run each batch as this many sub-batches on side streams (detect_packed), with results bit-identical to
        streams=1; a forward that calibrates the F16F8 scales runs unsplit, so that they come from the whole batch."""
        if mode is not None:
            planes = self.MODES[mode]
        self.graph_max_batch = int(graph_max_batch)
        self._graphs = {}
        if not torch.cuda.is_available():
            raise N.CtpnError("ctpn_b200.Engine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        torch.cuda.set_device(self.device)
        N.check(N.lib.ctpn_device_ok(device), "ctpn_device_ok")
        self.planes = int(planes)
        self.cfg = dict(DEFAULT_CFG)
        if cfg:
            self.cfg.update(cfg)
        h = C.c_void_p()
        N.check(N.lib.ctpn_net_create(C.byref(h), self.planes), "ctpn_net_create")
        self._net = h
        if conv_simt:          # float32 SIMT reference convolutions: only in the test library (CTPN_B200_LIB=dbg)
            N.check(N.lib.ctpn_net_set_option(self._net, b"conv_simt", 1), "set_option")
        if keep_activations:
            N.check(N.lib.ctpn_net_set_option(self._net, b"keep_activations", 1), "set_option")
        self._ws = {}
        self._pinned = {}
        self.streams = int(streams)
        self._side = []
        self._calibrated = False      # mirrors the library's F16F8 calibration state (see detect_packed)
        if weights is not None:
            self.load_weights(weights)

    def __del__(self):
        try:
            if getattr(self, "_net", None):
                N.lib.ctpn_net_destroy(self._net)
                self._net = None
        except Exception:
            pass

    # ---- weights -------------------------------------------------------------------------
    def load_weights(self, weights):
        """weights: dict TF-variable-name -> float32 ndarray (SURVEY.md App. A.2), or a path understood by
        load_weight_file: TF checkpoint (prefix or directory), frozen .pb, VGG16 .npy dict, .npz."""
        if isinstance(weights, str):
            weights = load_weight_file(weights)
        self._graphs.clear()          # captured graphs hold the old weight buffers' addresses
        self._calibrated = False      # new weights re-arm the F16F8 calibration
        for name, arr in weights.items():
            a = np.ascontiguousarray(arr, dtype=np.float32)
            N.check(N.lib.ctpn_net_set_weight(self._net, name.encode(), N.ptr(a), a.size), "ctpn_net_set_weight(%s)" % name)

    # ---- buffers ---------------------------------------------------------------------------
    def _workspace(self, key, nbytes):
        buf = self._ws.get(key)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=self.device)
            self._ws[key] = buf
        return buf

    def _pin(self, key, shape, dtype):
        key = (key, tuple(shape), dtype)       # one buffer per use AND shape: alternating shape buckets never re-pin
        t = self._pinned.get(key)
        if t is None:
            if len(self._pinned) >= 64:
                self._pinned.clear()
            t = torch.empty(tuple(shape), dtype=dtype, pin_memory=True)
            self._pinned[key] = t
        return t

    @staticmethod
    def feature_hw(H, W):
        fh, fw = C.c_int(), C.c_int()
        N.check(N.lib.ctpn_net_feature_hw(H, W, C.byref(fh), C.byref(fw)), "ctpn_net_feature_hw")
        return fh.value, fw.value

    def _sizes_device(self, sizes, B, H, W, least=16, what="sizes", device=None):
        """Per-image (h, w) of a ragged batch on its [B, H, W] canvas -> device int32 [B,2], checked on the host.
        device: a device int32 [B,2] tensor that already holds (or, in stream order, will hold) these sizes -- returned
        instead of uploading them, which costs a pageable copy and a stream synchronise per call."""
        s = sizes.cpu().numpy() if torch.is_tensor(sizes) else np.asarray(sizes)
        s = np.asarray(s, np.int64).reshape(-1, 2) if s.size else s.reshape(0, 2)
        if s.shape != (B, 2):
            raise ValueError("%s: expected %d (h, w) pairs, got shape %s" % (what, B, tuple(np.shape(sizes))))
        if (s[:, 0] > H).any() or (s[:, 1] > W).any() or (s < least).any():
            raise ValueError("%s: every (h, w) must lie within the %dx%d canvas and be at least %d" % (what, H, W, least))
        if device is not None:
            assert device.is_cuda and device.dtype == torch.int32 and tuple(device.shape) == (B, 2) and device.is_contiguous()
            return device
        return torch.from_numpy(s.astype(np.int32)).to(self.device, non_blocking=False)

    # ---- stages ----------------------------------------------------------------------------
    def forward_heads(self, images, ws_key="net", sizes=None, sizes_device=None):
        """images: CUDA tensor [B,H,W,3], uint8 BGR (mean subtraction fused) or float32 blob
        (already mean-subtracted, test.py:9).  Returns (rpn_cls_score [B,h,w,20] logits,
        rpn_bbox_pred [B,h,w,40]) float32 CUDA tensors.
        sizes: [B,2] (h, w) per image for a ragged batch (image b in rows < h and columns < w of its canvas slice, the rest
        ignored); each image's heads within (h >> 4, w >> 4) then equal a forward of that image alone.  None: uniform.
        sizes_device: the same sizes already on the device (see _sizes_device)."""
        assert images.is_cuda and images.dim() == 4 and images.shape[3] == 3 and images.is_contiguous()
        is_f32 = images.dtype == torch.float32
        assert is_f32 or images.dtype == torch.uint8
        B, H, W, _ = images.shape
        fh, fw = self.feature_hw(H, W)
        need = N.lib.ctpn_net_workspace_bytes(self._net, B, H, W)
        ws = self._workspace(ws_key, need)
        cls = torch.empty((B, fh, fw, 20), dtype=torch.float32, device=self.device)
        bbox = torch.empty((B, fh, fw, 40), dtype=torch.float32, device=self.device)
        if sizes is None:
            N.check(N.lib.ctpn_net_forward(self._net, N.ptr(images), int(is_f32), B, H, W, N.ptr(cls), N.ptr(bbox),
                                           N.ptr(ws), ws.numel(), N.stream_ptr()), "ctpn_net_forward")
        else:
            sz = self._sizes_device(sizes, B, H, W, device=sizes_device)
            N.check(N.lib.ctpn_net_forward_ragged(self._net, N.ptr(images), int(is_f32), N.ptr(sz), B, H, W, N.ptr(cls),
                                                  N.ptr(bbox), N.ptr(ws), ws.numel(), N.stream_ptr()), "ctpn_net_forward_ragged")
        self._calibrated = True
        return cls, bbox

    def recalibrate(self):
        """F16F8 mode: derive the activation scales again from the next batch (they are frozen after the first one).
        The scales put each layer's calibration maximum two binades below e4m3 saturation; activations beyond that saturate
        in the e4m3 copies, and those elements fall back to fp16 accuracy as long as they stay below 65504 / s in the fp16
        plane.  s is 1 unless the calibration maximum exceeds 2^14; a layer with s < 1 has only 2-3 binades of fp16 headroom,
        past which the element saturates in fp16 too and its error is unbounded.  So calibrate on representative images --
        not on a flat warm-up image -- and call this again when the input distribution changes."""
        N.check(N.lib.ctpn_net_set_option(self._net, b"recalibrate", 1), "set_option")
        self._calibrated = False
        self._graphs.clear()          # captured graphs hold the old scales as kernel arguments

    def tap(self, name):
        """Debug: float32 copy of a named activation of the last forward (keep_activations=True)."""
        cnt = C.c_size_t()
        N.check(N.lib.ctpn_net_debug_tap(self._net, name.encode(), None, 0, C.byref(cnt), None), "debug_tap")
        out = torch.empty(cnt.value, dtype=torch.float32, device=self.device)
        N.check(N.lib.ctpn_net_debug_tap(self._net, name.encode(), N.ptr(out), out.numel(), C.byref(cnt), N.stream_ptr()), "debug_tap")
        return out

    def proposals(self, cls, bbox, im_info, cls_is_logit=True, cfg=None, ws_key="prop", out=None, feat_sizes=None,
                  feat_sizes_device=None):
        """Batched proposal layer (proposal_layer_tf.py:14-157) on CUDA tensors.
        Returns rois [B,post,5] (score,x1,y1,x2,y2), index [B,post] int32, count [B] int32.
        out=(rois, count): write into these (contiguous) tensors instead of allocating.
        feat_sizes: [B,2] (fh, fw) per image of a ragged batch: only those cells of each image's heads are read, and index is
        image-local ((h * fw + w) * 10 + a).  None: every cell.  feat_sizes_device: feat_sizes already on the device (see
        _sizes_device)."""
        c = dict(self.cfg)
        if cfg:
            c.update(cfg)
        B, H, W, _ = cls.shape
        pre, post = int(c["RPN_PRE_NMS_TOP_N"]), int(c["RPN_POST_NMS_TOP_N"])
        NA = H * W * 10
        max_n = pre if 0 < pre < NA else NA
        rows = post if post > 0 else max_n
        need = N.lib.ctpn_proposals_workspace_bytes(B, H, W, pre)
        ws = self._workspace(ws_key, need)
        if out is not None:
            rois, count = out
            assert rois.shape == (B, rows, 5) and count.shape == (B,) and rois.is_contiguous() and count.is_contiguous()
        else:
            rois = torch.empty((B, rows, 5), dtype=torch.float32, device=self.device)
            count = torch.empty((B,), dtype=torch.int32, device=self.device)
        index = torch.empty((B, rows), dtype=torch.int32, device=self.device)
        im_info = im_info.to(device=self.device, dtype=torch.float32).contiguous()
        if feat_sizes is not None:
            fs = self._sizes_device(feat_sizes, B, H, W, least=1, what="feat_sizes", device=feat_sizes_device)
            N.check(N.lib.ctpn_proposals_ragged(N.ptr(cls.contiguous()), int(cls_is_logit), N.ptr(bbox.contiguous()), N.ptr(im_info),
                                                N.ptr(fs), B, H, W, int(c["FEAT_STRIDE"]), pre, post, float(c["RPN_NMS_THRESH"]),
                                                float(c["RPN_MIN_SIZE"]), int(bool(c["ANCHORS_PY2"])), N.ptr(rois), N.ptr(index),
                                                N.ptr(count), N.ptr(ws), ws.numel(), N.stream_ptr()), "ctpn_proposals_ragged")
            return rois, index, count
        N.check(N.lib.ctpn_proposals(N.ptr(cls.contiguous()), int(cls_is_logit), N.ptr(bbox.contiguous()), N.ptr(im_info),
                                     B, H, W, int(c["FEAT_STRIDE"]), pre, post, float(c["RPN_NMS_THRESH"]),
                                     float(c["RPN_MIN_SIZE"]), int(bool(c["ANCHORS_PY2"])), N.ptr(rois), N.ptr(index),
                                     N.ptr(count), N.ptr(ws), ws.numel(), N.stream_ptr()), "ctpn_proposals")
        return rois, index, count

    # ---- public API ------------------------------------------------------------------------
    def result_rows(self):
        rows = int(self.cfg["RPN_POST_NMS_TOP_N"])
        if rows <= 0:
            raise ValueError("the packed result path needs RPN_POST_NMS_TOP_N > 0 (use Engine.proposals for an uncapped proposal list)")
        return rows

    @staticmethod
    def unpack(packed, B, rows):
        """Views (rois [..,B,rows,5] f32, count [..,B] i32) of packed result buffers [.., B*rows*5 + B] (torch or numpy)."""
        n = B * rows * 5
        lead = tuple(packed.shape[:-1])
        rois = packed[..., :n].reshape(lead + (B, rows, 5))
        tail = packed[..., n:]
        count = tail.view(torch.int32) if torch.is_tensor(tail) else tail.view(np.int32)
        return rois, count

    def detect_packed(self, images, im_info, ws_tag="", sizes=None, device_sizes=None):
        """images: CUDA [B,H,W,3] uint8/float32; im_info: [B,3] tensor (blob_h, blob_w, scale).
        Returns ONE float32 device buffer [B*post*5 + B]: the rois of all images followed by the int32 counts
        (bit pattern), so that the D2H / the multi-GPU gather of a batch's results is a single transfer.
        sizes: [B,2] (h, w) per image of a ragged batch (see forward_heads), or None.  device_sizes: (sizes, sizes >> 4) as
        device int32 [B,2] tensors, when the caller has uploaded them with the batch (see _sizes_device)."""
        B = int(images.shape[0])
        sz_d, feat_d = device_sizes if device_sizes is not None else (None, None)
        if sizes is not None:
            sizes = np.asarray(sizes.cpu() if torch.is_tensor(sizes) else sizes, np.int64).reshape(-1, 2)
            feat = sizes >> 4
        rows = self.result_rows()
        packed = torch.empty(B * rows * 5 + B, dtype=torch.float32, device=self.device)
        rois, count = self.unpack(packed, B, rows)
        # a forward that calibrates the F16F8 scales runs unsplit: the scales must come from the whole batch, as with streams=1
        n = min(self.streams, B) if self._calibrated or self.planes != self.MODES["f16f8"] else 1
        if n <= 1:
            cls, bbox = self.forward_heads(images, ws_key="net" + ws_tag, sizes=sizes, sizes_device=sz_d)
            self.proposals(cls, bbox, im_info, cls_is_logit=True, ws_key="prop" + ws_tag, out=(rois, count),
                           feat_sizes=None if sizes is None else feat, feat_sizes_device=feat_d)
            return packed
        # sub-batches on side streams: the SIMT kernels of one sub-batch (conv1_1, BiLSTM, sort, NMS) run beside
        # the tensor-core kernels of the other (a persistent conv CTA leaves room for them on every SM)
        main = torch.cuda.current_stream()
        if len(self._side) < n:
            self._side = [torch.cuda.Stream(device=self.device) for _ in range(n)]
        im_info = im_info.to(self.device)
        bounds = [B * i // n for i in range(n + 1)]
        for i in range(n):
            st = self._side[i]
            st.wait_stream(main)
            with torch.cuda.stream(st):
                lo, hi = bounds[i], bounds[i + 1]
                cls, bbox = self.forward_heads(images[lo:hi], ws_key="net%d" % i, sizes=None if sizes is None else sizes[lo:hi],
                                               sizes_device=None if sz_d is None else sz_d[lo:hi])
                self.proposals(cls, bbox, im_info[lo:hi], cls_is_logit=True, ws_key="prop%d" % i, out=(rois[lo:hi], count[lo:hi]),
                               feat_sizes=None if sizes is None else feat[lo:hi],
                               feat_sizes_device=None if feat_d is None else feat_d[lo:hi])
        for st in self._side[:n]:
            main.wait_stream(st)
        return packed

    def detect_packed_graphed(self, images, im_info):
        """detect_packed through a CUDA graph captured once per (shape, dtype) bucket: inputs are copied into the graph's
        static buffers, the whole kernel sequence (conv stack, BiLSTM, heads, proposal layer) is replayed with one launch,
        and the result is the graph's static packed buffer (valid until the next call for the same bucket).  Used for small
        batches, where launch overhead dominates; the first two calls of a bucket run eagerly (weight upload, F16F8
        calibration, attribute / tensor-map caches must be warm before a capture)."""
        key = (tuple(images.shape), images.dtype)
        g = self._graphs.get(key)
        if g is None:
            g = self._graphs[key] = {"calls": 0}
        if "graph" not in g:
            g["calls"] += 1
            if g["calls"] <= 2 or self.streams > 1:
                return self.detect_packed(images, im_info)
            g["in"] = torch.empty_like(images)
            g["info"] = torch.empty((images.shape[0], 3), dtype=torch.float32, device=self.device)
            g["in"].copy_(images)
            g["info"].copy_(im_info)
            torch.cuda.current_stream().synchronize()
            graph = torch.cuda.CUDAGraph()
            tag = "/graph%d" % len([1 for v in self._graphs.values() if "graph" in v])
            self.detect_packed(g["in"], g["info"], ws_tag=tag)      # allocates this bucket's OWN workspaces (never resized or
            torch.cuda.current_stream().synchronize()               # shared: the graph holds their addresses)
            with torch.cuda.graph(graph):
                g["out"] = self.detect_packed(g["in"], g["info"], ws_tag=tag)
            g["graph"] = graph
        g["in"].copy_(images, non_blocking=True)
        g["info"].copy_(im_info, non_blocking=True)
        g["graph"].replay()
        return g["out"]

    def detect_device(self, images, im_info):
        """As detect_packed; returns device tensors (rois [B,post,5], count [B]) -- views of the packed buffer."""
        return self.unpack(self.detect_packed(images, im_info), int(images.shape[0]), self.result_rows())

    def all_gather(self, rois, count):
        """Multi-GPU (one process per GPU, torch.distributed/NCCL initialised by the caller): every rank
        contributes the fixed-shape results of its image shard; returns ([world*B,post,5], [world*B])
        ordered by rank.  The only collective on the path (images are independent)."""
        from .dist import gather_results
        return gather_results(rois, count)

    def _stage_host(self, images, slot=0):
        """Host batch (ndarray / CPU tensor) -> pinned tensor.  A pinned tensor passes through; anything else is copied
        into the pinned staging buffer of `slot` (callers that keep two transfers in flight alternate slots and wait
        for the slot's previous H2D before calling)."""
        if isinstance(images, torch.Tensor):
            assert images.device.type == "cpu" and images.dtype in (torch.uint8, torch.float32)
            src = images.contiguous()
            if src.is_pinned():
                return src
            pinned = self._pin(("in", slot), tuple(src.shape), src.dtype)
            pinned.copy_(src)
            return pinned
        arr = np.ascontiguousarray(images)
        dt = torch.uint8 if arr.dtype == np.uint8 else torch.float32
        pinned = self._pin(("in", slot), arr.shape, dt)
        pinned.numpy()[...] = arr if dt == torch.uint8 else arr.astype(np.float32, copy=False)
        return pinned

    def _split_results(self, packed_h, B, rows):
        """Pinned packed results [.., B*rows*5+B] -> list of per-image [n,5] arrays (rank order, image order)."""
        rois, count = self.unpack(packed_h.numpy(), B, rows)
        rois = rois.reshape(-1, rows, 5)
        count = count.reshape(-1)
        return [rois[i, :int(count[i])].copy() for i in range(rois.shape[0])]

    def rois_batch(self, images, im_info=None, gather=False):
        """images: host ndarray, (pinned) CPU tensor or device tensor [B,H,W,3] (uint8 BGR, or float32 mean-subtracted blob);
        im_info: [B,3] (defaults to (H, W, 1.0)).  Returns one float32 [n,5] array per image,
        rows (score, x1, y1, x2, y2) in blob coordinates -- the 'rois' tensor of the reference
        graph (network.py:217).  H2D of the inputs and D2H of the results are part of the call.
        gather=True (multi-GPU): results of all ranks' shards, in rank order."""
        if isinstance(images, torch.Tensor) and images.device.type == "cuda":
            # already resident (e.g. the output of resize_images): no staging, no H2D
            assert images.dtype in (torch.uint8, torch.float32)
            stage = images.contiguous()
        else:
            stage = self._stage_host(images)
        B, H, W, _ = stage.shape
        if im_info is None:
            im_info = np.array([[H, W, 1.0]] * B, np.float32)
        info_h = self._pin("info", (B, 3), torch.float32)
        info_h.numpy()[...] = np.asarray(im_info, np.float32).reshape(B, 3)
        dev = stage.to(self.device, non_blocking=True)
        info_d = info_h.to(self.device, non_blocking=True)
        if 0 < B <= self.graph_max_batch and not gather:
            packed = self.detect_packed_graphed(dev, info_d)
        else:
            packed = self.detect_packed(dev, info_d)
        if gather:
            from .dist import gather_packed
            packed = gather_packed(packed)
        out_h = self._pin("out", tuple(packed.shape), torch.float32)
        out_h.copy_(packed, non_blocking=True)       # one D2H: rois and counts travel together
        torch.cuda.current_stream().synchronize()
        return self._split_results(out_h, B, self.result_rows())

    def rois_batches(self, batches, im_info=None, gather=False):
        """Pipelined version of rois_batch for a stream of equally shaped host batches (pinned uint8/float32 CPU tensors
        or ndarrays).  Three stages overlap: the H2D copy of batch k+1 (copy stream), the compute of batch k (current
        stream), and the multi-GPU gather (gather=True: one all-gather of the packed results) + D2H of batch k-1's
        results (result stream).  The host blocks only on the event of the batch it is about to yield, after the next
        batch's work has been enqueued, so the GPU never waits for Python.  Yields the rois_batch() result of every
        batch in order."""
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
            self._result_stream = torch.cuda.Stream(device=self.device)
        copy_stream, result_stream = self._copy_stream, self._result_stream
        main = torch.cuda.current_stream()
        rows = self.result_rows()
        bufs = self.__dict__.setdefault("_stream_bufs", {})   # two persistent device input buffers, used alternately
        computed = [None, None]    # event: the compute that read device buffer `slot` has finished
        copied = [None, None]      # event: the H2D out of pinned staging buffer `slot` has finished
        counter = [0]

        def stage(images):
            slot = counter[0] & 1
            counter[0] += 1
            if copied[slot] is not None:
                copied[slot].synchronize()           # the staging buffer of this slot is free again (ADVICE r1: host race)
            src = self._stage_host(images, slot)
            key = (slot, tuple(src.shape), src.dtype)
            if key not in bufs:
                # A fresh block from the caching allocator may be memory that tensors of the compute stream have just
                # released while their kernels are still running: writing it from the copy stream would race with them
                # (seen as a corrupted first image of the second batch).  Allocate in the copy stream's pool and let the
                # copy stream catch up with the compute stream once, at creation; the buffer then lives as long as the engine.
                with torch.cuda.stream(copy_stream):
                    copy_stream.wait_stream(main)
                    bufs[key] = torch.empty(tuple(src.shape), dtype=src.dtype, device=self.device)
            dev = bufs[key]
            with torch.cuda.stream(copy_stream):
                if computed[slot] is not None:
                    copy_stream.wait_event(computed[slot])     # the previous user of this device buffer has finished
                dev.copy_(src, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(copy_stream)
            copied[slot] = ev
            return dev, ev, slot

        def finish(pending):
            out_h, ev, B, keep = pending
            ev.synchronize()
            del keep
            return self._split_results(out_h, B, rows)

        it = iter(batches)
        try:
            nxt = stage(next(it))
        except StopIteration:
            return
        pending = None
        k = 0
        while nxt is not None:
            dev, ev, slot = nxt
            B, H, W, _ = dev.shape
            info = im_info if im_info is not None else np.array([[H, W, 1.0]] * B, np.float32)
            info_h = self._pin(("info", k & 1), (B, 3), torch.float32)
            info_h.numpy()[...] = np.asarray(info, np.float32).reshape(B, 3)
            main.wait_event(ev)
            packed = self.detect_packed(dev, info_h.to(self.device, non_blocking=True))
            done = torch.cuda.Event()
            done.record(main)
            computed[slot] = done
            with torch.cuda.stream(result_stream):
                result_stream.wait_event(done)
                res = packed
                if gather:
                    from .dist import gather_packed
                    res = gather_packed(packed)
                out_h = self._pin(("out", k & 1), tuple(res.shape), torch.float32)
                out_h.copy_(res, non_blocking=True)
                rev = torch.cuda.Event()
                rev.record(result_stream)
            this = (out_h, rev, B, (packed, res))
            try:
                nxt = stage(next(it))          # H2D of the next batch: overlaps the compute enqueued above
            except StopIteration:
                nxt = None
            if pending is not None:
                yield finish(pending)          # blocks on batch k-1 while batch k is already queued on the GPU
            pending = this
            k += 1
        if pending is not None:
            yield finish(pending)

    def detect_lines_batches(self, batches, mode="H", im_info=None, workers=8, gather=False, cfg=None, im_hw=None):
        """The whole ctpn() call chain (demo.py:55-68 minus file I/O) for a stream of host batches: rois_batches() on the
        GPU, then TextDetector.detect of every image in the library's host connector (ctpn_text_lines_host, which
        releases the GIL) on a pool of `workers` threads, one batch behind the GPU.  With gather=True (multi-GPU) the rois of
        all ranks are gathered as in rois_batches and every rank runs the connector on its own shard.  Yields, per batch, a list of
        float64 [m,9] text-line arrays (x1,y1,x2,y2,x3,y3,x4,y4,score) in the frame im_hw = (h, w) of the image the blobs were
        made from (resize_im's output): text_lines(rois[:, 1:5] / np.float64(scale), rois[:, 0], im_hw, mode, cfg), as
        test_ctpn and TextDetector compute them, with the scale im_info[0, 2] as given (pass im_info as float64 to keep an
        inexact scale such as 1000 / 1100 exactly as test_ctpn has it).  im_hw=None: the frame is each batch's (H, W), which
        needs scale 1 -- the blob's size divided by the scale does not give the image's size back in general."""
        from concurrent.futures import ThreadPoolExecutor
        from .textlines import text_lines

        scale = 1.0 if im_info is None else float(np.asarray(im_info).reshape(-1, 3)[0, 2])
        if im_hw is None and scale != 1.0:
            raise ValueError("detect_lines_batches: im_hw= (the frame of the lines) is needed when the scale is not 1 (got %r)" % scale)
        frame = None if im_hw is None else tuple(int(v) for v in im_hw)
        if frame is not None and len(frame) != 2:
            raise ValueError("detect_lines_batches: im_hw must be one (h, w) pair (got %r)" % (im_hw,))

        def lines_of(rois, size):
            return text_lines(rois[:, 1:5] / np.float64(scale), rois[:, 0], size, mode, cfg)

        batches = iter(batches)
        shapes = []

        def tracked():
            for b in batches:
                shapes.append(tuple(b.shape[1:3]))
                yield b

        pool = getattr(self, "_line_pool", None)
        if pool is None or pool._max_workers != workers:
            pool = self._line_pool = ThreadPoolExecutor(max_workers=workers, thread_name_prefix="ctpn-lines")
        shard = None
        if gather:
            import torch.distributed as dist
            shard = (dist.get_rank(), dist.get_world_size())
        pending = None
        for k, rois_list in enumerate(self.rois_batches(tracked(), im_info=im_info, gather=gather)):
            if shard is not None:      # every rank holds all ranks' rois after the gather; each builds the lines of its own shard
                per = len(rois_list) // shard[1]
                rois_list = rois_list[shard[0] * per:(shard[0] + 1) * per]
            size = shapes[k] if frame is None else frame
            futs = [pool.submit(lines_of, r, size) for r in rois_list]
            if pending is not None:
                yield [f.result() for f in pending]
            pending = futs
        if pending is not None:
            yield [f.result() for f in pending]

    def detect_batch(self, images, im_scale=1.0):
        """Returns a list of (scores [n] f32, boxes [n,4] f32) per image, boxes divided by
        im_scale exactly as lib/fast_rcnn/test.py:54-57 does."""
        B, H, W, _ = images.shape
        info = np.array([[H, W, im_scale]] * B, np.float32)
        return [(r[:, 0], r[:, 1:5] / np.float32(im_scale)) for r in self.rois_batch(images, info)]

    def detect_list(self, images, max_batch=32):
        """Mixed-shape input (BASELINE.json configs[4]): a list of HxWx3 images of arbitrary sizes is grouped
        into shape buckets, every bucket runs as batches of up to `max_batch`, and the (scores, boxes) results
        come back in the order of the input list.  Images are taken at scale 1 (use test_ctpn for the
        reference's rescaling rules)."""
        buckets = {}
        for i, im in enumerate(images):
            buckets.setdefault((im.shape, im.dtype.str), []).append(i)
        out = [None] * len(images)
        for (_shape, _dt), idxs in buckets.items():
            for k in range(0, len(idxs), max_batch):
                part = idxs[k:k + max_batch]
                res = self.detect_batch(np.stack([images[i] for i in part]))
                for i, r in zip(part, res):
                    out[i] = r
        return out

    def detect_ragged(self, images, im_scales=None, max_batch=32):
        """Images of different sizes in shared batches: a list of HxWx3 uint8 BGR images or float32 mean-subtracted blobs
        (H, W >= 16), with im_scales[i] the scale that made image i (default 1).  ragged_plan() groups them into batches of
        at most `max_batch` on a canvas of each batch's largest H and W; every image is computed as if it ran alone
        (ctpn_net_forward_ragged), with im_info (h, w, im_scale) of its own.  Returns [(scores, boxes / im_scale)] in input
        order, as detect_batch returns them.  Raises ValueError on a bad image or scale list."""
        scales = [1.0] * len(images) if im_scales is None else list(im_scales)
        rois = self.rois_ragged(images, im_scales, max_batch)
        return [(r[:, 0], r[:, 1:5] / np.float32(s)) for r, s in zip(rois, scales)]

    def rois_ragged(self, images, im_scales=None, max_batch=32):
        """detect_ragged's rois: one float32 [n,5] array (score, x1, y1, x2, y2) in blob coordinates per image, in input
        order (test_ctpn divides these by its float64 im_scale; detect_batch by float32)."""
        images = list(images)
        n = len(images)
        scales = [1.0] * n if im_scales is None else [float(s) for s in im_scales]
        if len(scales) != n:
            raise ValueError("detect_ragged: %d images but %d scales" % (n, len(scales)))
        arrs, shapes, dtypes = [], [], []
        for i, im in enumerate(images):
            a = im.numpy() if torch.is_tensor(im) else np.asarray(im)
            if a.ndim != 3 or a.shape[2] != 3 or a.dtype not in (np.uint8, np.float32):
                raise ValueError("detect_ragged: image %d must be HxWx3 uint8 or float32 (got %s %s)" % (i, a.shape, a.dtype))
            if a.shape[0] < 16 or a.shape[1] < 16:
                raise ValueError("detect_ragged: image %d is %dx%d; both sides must be at least 16" % (i, a.shape[0], a.shape[1]))
            arrs.append(a)
            shapes.append((int(a.shape[0]), int(a.shape[1])))
            dtypes.append(a.dtype.str)
        out = [None] * n
        rows = self.result_rows()
        for idxs, (H, W) in ragged_plan(shapes, dtypes, max_batch):
            B = len(idxs)
            dt = torch.uint8 if arrs[idxs[0]].dtype == np.uint8 else torch.float32
            canvas = self._pin("ragged", (B, H, W, 3), dt)        # padding keeps whatever it held: the kernels never read it
            cn = canvas.numpy()
            for k, i in enumerate(idxs):
                h, w = shapes[i]
                cn[k, :h, :w] = arrs[i]
            info_h = self._pin("info", (B, 3), torch.float32)
            info_h.numpy()[...] = [[shapes[i][0], shapes[i][1], scales[i]] for i in idxs]
            sizes = np.array([shapes[i] for i in idxs], np.int64)
            packed = self.detect_packed(canvas.to(self.device, non_blocking=True), info_h.to(self.device, non_blocking=True),
                                        sizes=sizes)
            out_h = self._pin("out", tuple(packed.shape), torch.float32)
            out_h.copy_(packed, non_blocking=True)
            torch.cuda.current_stream().synchronize()              # also frees the pinned canvas for the next batch
            for i, r in zip(idxs, self._split_results(out_h, B, rows)):
                out[i] = r
        return out

    def resize_images(self, images, fx, fy=None):
        """cv2.resize(im, None, None, fx=fx, fy=fy, interpolation=cv2.INTER_LINEAR) of a uint8 batch [B,H,W,C] on the
        device (bit-exact with OpenCV; resize_im of ctpn/demo.py:21-25).  images: ndarray or torch tensor (host or
        device); returns a uint8 device tensor [B,dh,dw,C]."""
        fy = fx if fy is None else fy
        t = images if torch.is_tensor(images) else torch.from_numpy(np.ascontiguousarray(images))
        if t.dtype != torch.uint8 or t.dim() != 4:
            raise ValueError("resize_images expects a uint8 [B,H,W,C] batch")
        t = t.to(self.device, non_blocking=True).contiguous()
        B, H, W, Cn = t.shape
        dh, dw = C.c_int(0), C.c_int(0)
        N.check(N.lib.ctpn_resize_out_size(H, W, float(fx), float(fy), C.byref(dh), C.byref(dw)), "ctpn_resize_out_size")
        out = torch.empty((B, dh.value, dw.value, Cn), dtype=torch.uint8, device=self.device)
        N.check(N.lib.ctpn_resize_linear_u8(N.ptr(t), B, H, W, Cn, float(fx), float(fy), N.ptr(out), dh.value, dw.value,
                                            N.stream_ptr()), "ctpn_resize_linear_u8")
        return out

    def _mean_lut(self):
        """Device float32 [256,3]: float32(double(v) - PIXEL_MEANS[c]), the mean subtraction of _get_image_blob."""
        if getattr(self, "_lut", None) is None:
            means = np.array([102.9801, 115.9465, 122.7717])              # cfg.PIXEL_MEANS (config.py:200), BGR
            self._lut = torch.from_numpy((np.arange(256, dtype=np.float64)[:, None] - means[None, :]).astype(np.float32)).to(self.device)
        return self._lut

    def image_blob(self, images, im_scale):
        """_get_image_blob (lib/fast_rcnn/test.py:7-31) on the device for a same-shape uint8 BGR batch [B,H,W,3]: mean
        subtraction (float32(double(v) - PIXEL_MEANS)) fused with the float32 cv2.resize by im_scale.  Returns a float32
        device blob [B,dh,dw,3], bit-exact with OpenCV's own float INTER_LINEAR code (IPP-dispatching cv2 builds differ
        from that by up to ~1e-2 on 8-bit-range data; see csrc/resize.cu)."""
        t = images if torch.is_tensor(images) else torch.from_numpy(np.ascontiguousarray(images))
        if t.dtype != torch.uint8 or t.dim() != 4 or t.shape[3] != 3:
            raise ValueError("image_blob expects a uint8 [B,H,W,3] batch")
        t = t.to(self.device, non_blocking=True).contiguous()
        B, H, W, _ = t.shape
        self._mean_lut()
        dh, dw = C.c_int(0), C.c_int(0)
        N.check(N.lib.ctpn_resize_out_size(H, W, float(im_scale), float(im_scale), C.byref(dh), C.byref(dw)), "ctpn_resize_out_size")
        out = torch.empty((B, dh.value, dw.value, 3), dtype=torch.float32, device=self.device)
        N.check(N.lib.ctpn_image_blob_f32(N.ptr(t), N.ptr(self._lut), B, H, W, float(im_scale), float(im_scale), N.ptr(out),
                                          dh.value, dw.value, N.stream_ptr()), "ctpn_image_blob_f32")
        return out

    def detect_scaled(self, images):
        """test_ctpn() for a same-shape uint8 batch with the reference's rescaling rule on the device: im_scale =
        SCALES[0] / short side, capped so that the long side stays within MAX_SIZE (test.py:13-20); scale 1 takes the
        uint8 fast path, anything else image_blob().  Returns [(scores, boxes)] with boxes divided by im_scale (test.py:54-57)."""
        H, W = int(images.shape[1]), int(images.shape[2])
        target, max_size = float(self.cfg["SCALES"][0]), float(self.cfg["MAX_SIZE"])
        im_scale = target / min(H, W)
        if np.round(im_scale * max(H, W)) > max_size:
            im_scale = max_size / max(H, W)
        if im_scale == 1.0:
            return self.detect_batch(images, 1.0)
        blob = self.image_blob(images, im_scale)
        info = np.array([[blob.shape[1], blob.shape[2], im_scale]] * blob.shape[0], np.float32)
        return [(r[:, 0], r[:, 1:5] / np.float32(im_scale)) for r in self.rois_batch(blob, info)]

    def detect_resized(self, images, scale=600, max_scale=1200):
        """The front half of ctpn() (demo.py:59-61) for a same-shape uint8 batch: resize_im on the device (short side
        -> scale, long side <= max_scale), then the detector.  Returns ([(scores, boxes)], f); boxes are in the resized
        frame, as TextDetector expects them (draw_boxes divides by f).  Assumes the resized long side is within
        cfg.TEST.MAX_SIZE so that _get_image_blob adds no second rescale (true for the default 600 / 1200 / 1000
        settings whenever the aspect ratio is <= 5:3)."""
        H, W = int(images.shape[1]), int(images.shape[2])
        f = float(scale) / min(H, W)
        if max_scale is not None and f * max(H, W) > max_scale:
            f = float(max_scale) / max(H, W)
        resized = images if f == 1.0 else self.resize_images(images, f)
        return self.detect_batch(resized), f

    def rois_images(self, images, resize=True, max_batch=32, return_resized=False, scale=600, max_scale=1200, channels="BGR"):
        """The front half of ctpn() (demo.py:59-61) plus test_ctpn for a list of raw HxWx3 uint8 BGR images of any sizes,
        front-end on the device: resize_im (short side -> scale, long side <= max_scale; resize=False: the images are
        already at that scale) and _get_image_blob (uint8 when im_scale == 1, else the mean-subtracted float32 rescale),
        then ragged batches of at most max_batch (frontend_plan + ragged_plan).  Each batch's sources travel in one pinned
        H2D copy; ctpn_resize_linear_u8_ragged writes the uint8 canvas (or, for float32 batches, a uint8 canvas that
        ctpn_image_blob_f32_ragged turns into the float32 blob canvas), and detect_packed runs the batch with per-image
        extents.  Returns, in input order, (rois float32 [n,5] in blob coordinates, im_scale, f) per image -- and the
        resize_im output as a host uint8 array as a 4th item with return_resized (what draw_boxes draws on).  Every image
        is bit-identical to the host front-end with OpenCV's own code (IPP-dispatching cv2 builds differ on float
        rescales) followed by detect on that image alone.  Raises ValueError on a bad image (see frontend_plan).

        The images may instead all be CUDA uint8 [H, W, 3] tensors on this engine's device, at any strides (crop views,
        chw.permute(1, 2, 0), zero strides): ctpn_resize_linear_u8_strided reads them in place, so no image crosses the
        bus, and the results equal those of the same call on host copies.  They must be ready on the stream that is current
        when the call is made (torch's rule); the engine synchronises nothing for them.  A list that mixes host images and
        CUDA tensors, or a tensor on another device, raises ValueError before any device work.  channels="RGB": every image
        of the call holds RGB (as torchvision decodes it) -- host images are flipped inside the packing copy, tensors are
        read through a negative channel stride.

        Or the images may all be YUV420 frames (video frames: NV12, NV21, I420, YV12 planes) on this engine's device:
        ctpn_resize_linear_u8_yuv420 reads the planes in place and converts each sample as cv2.cvtColor does, so the results
        equal those of the same call on cv2.cvtColor(frame, COLOR_YUV2BGR_*) -- return_resized included.  The stream rule
        above applies to the planes; a frame with odd sides, a plane on another device or channels="RGB" raises ValueError
        before any device work."""
        out = [None] * len(images)
        rows = self.result_rows()
        for idxs, items, out_h, resized, _, _, _ in self._images_batches(images, resize, max_batch, return_resized, scale,
                                                                         max_scale, "rois_images", channels=channels):
            for k, (i, r) in enumerate(zip(idxs, self._split_results(out_h, len(idxs), rows))):
                out[i] = (r, items[k].im_scale, items[k].f) + ((resized[k],) if return_resized else ())
        return out

    def _images_batches(self, images, resize, max_batch, return_resized, scale, max_scale, what, after=None, channels="BGR"):
        """The batches of rois_images / detect_lines_images.  Per ragged batch: front-end, network and proposal layer on the
        device (detect_packed's buffer), then after(packed, items) -- device work enqueued on the rois, returning the buffer
        to bring back (None: the packed rois themselves) -- and one D2H of that buffer.  Yields (input indices, their
        FrontendSteps, the pinned host copy, the resize_im outputs or None, the uint8 resize_im canvas, the device buffer
        brought back, a callable giving the batch's sources for source crops (line_crop_sources)); the pinned copy is reused
        by the next batch, and the canvas and the uploaded sources are rewritten by the next batch's work on the current
        stream.
        Host images go up in one pinned H2D per batch; CUDA tensors (images_on_device) are read in place by
        ctpn_resize_linear_u8_strided."""
        if not 1 <= int(max_batch) <= 64:
            raise ValueError("%s: max_batch must be 1..64 (the ragged front-end kernels take up to 64 images)" % what)
        check_channels(channels, what)
        images = list(images)
        device_images = images_on_device(images, self.device, what, channels)
        if not device_images:
            images = [im.numpy() if torch.is_tensor(im) else np.asarray(im) for im in images]
        plan = frontend_plan(images, resize=resize, scale=scale, max_scale=max_scale, cfg=self.cfg)
        lut = self._mean_lut()
        stream = N.stream_ptr()
        for idxs, (H, W) in ragged_plan([p.blob for p in plan], [p.dtype for p in plan], max_batch):
            B = len(idxs)
            items = [plan[i] for i in idxs]
            is_u8 = items[0].dtype == "|u1"
            if is_u8:          # im_scale == 1: resize_im writes the network's uint8 canvas directly
                u8 = canvas = torch.empty((B, H, W, 3), dtype=torch.uint8, device=self.device)
                Hr, Wr = H, W
            else:
                Hr, Wr = max(p.resized[0] for p in items), max(p.resized[1] for p in items)
                u8 = self._workspace("frontend_u8", B * Hr * Wr * 3)[:B * Hr * Wr * 3].view(B, Hr, Wr, 3)
                canvas = torch.empty((B, H, W, 3), dtype=torch.float32, device=self.device)
            resized_hw = np.array([p.resized for p in items], np.int32)
            fxy = np.array([[p.f, p.f] for p in items], np.float64)
            batch_images = [images[i] for i in idxs]
            if device_images:      # read in place: no staging, no image H2D
                resize_in_place(batch_images, device_images, channels, fxy, resized_hw, u8, stream)
                sources = functools.partial(line_crop_sources, batch_images, device_images, channels)
            else:
                nbytes = [images[i].size for i in idxs]
                offsets = np.cumsum([0] + nbytes[:-1]).astype(np.int64)
                total = int(sum(nbytes))
                pinned = self._pin("frontend_src", (1 << max(20, (total - 1).bit_length()),), torch.uint8)   # grow-only sizes
                pn = pinned.numpy()
                for k, i in enumerate(idxs):
                    h, w = images[i].shape[:2]
                    pn[offsets[k]:offsets[k] + nbytes[k]].reshape(h, w, 3)[...] = as_bgr(images[i], channels)
                src = self._workspace("frontend_src", total)
                src[:total].copy_(pinned[:total], non_blocking=True)           # the batch's one H2D
                hwp = np.array([images[i].shape[:2] + (images[i].shape[1],) for i in idxs], np.int32)
                N.check(N.lib.ctpn_resize_linear_u8_ragged(N.ptr(src), total, N.ptr(offsets), N.ptr(hwp), N.ptr(fxy),
                                                           N.ptr(resized_hw), B, 3, N.ptr(u8), Hr, Wr, stream),
                        "ctpn_resize_linear_u8_ragged")
                sources = functools.partial(line_crop_sources, batch_images, HOST, "BGR", src, offsets)
            if not is_u8:
                boffs = np.arange(B, dtype=np.int64) * (Hr * Wr * 3)
                bhwp = np.concatenate([resized_hw, np.full((B, 1), Wr, np.int32)], axis=1)
                bfxy = np.array([[p.im_scale, p.im_scale] for p in items], np.float64)
                blob_hw = np.array([p.blob for p in items], np.int32)
                N.check(N.lib.ctpn_image_blob_f32_ragged(N.ptr(u8), B * Hr * Wr * 3, N.ptr(boffs), N.ptr(bhwp), N.ptr(bfxy),
                                                         N.ptr(blob_hw), N.ptr(lut), B, N.ptr(canvas), H, W, stream),
                        "ctpn_image_blob_f32_ragged")
            info_h = self._pin("info", (B, 3), torch.float32)
            info_h.numpy()[...] = [[p.blob[0], p.blob[1], p.im_scale] for p in items]
            packed = self.detect_packed(canvas, info_h.to(self.device, non_blocking=True), sizes=np.array([p.blob for p in items]))
            result = packed if after is None else after(packed, items)
            out_h = self._pin("out", tuple(result.shape), result.dtype)
            out_h.copy_(result, non_blocking=True)
            resized = [u8[k, :p.resized[0], :p.resized[1]].cpu().numpy() for k, p in enumerate(items)] if return_resized else None
            torch.cuda.current_stream().synchronize()              # also frees the pinned sources for the next batch
            yield idxs, items, out_h, resized, u8, result, sources

    # ---- text lines on the device ----------------------------------------------------------
    @staticmethod
    def unpack_lines(packed, B, rows):
        """Views (lines [B,rows,9] f64, num [B] i32, status [B] i32) of a packed text-line buffer [B*rows*9 + B] float64
        (torch or numpy): the lines of all images followed by the int32 line counts and statuses (bit pattern)."""
        n = B * rows * 9
        lines = packed[:n].reshape(B, rows, 9)
        tail = packed[n:]
        t = tail.view(torch.int32) if torch.is_tensor(tail) else tail.view(np.int32)
        return lines, t[:B], t[B:2 * B]

    def text_lines(self, rois, count, im_hw, im_scales, mode="H", cfg=None, out=None, ws_key="lines"):
        """TextDetector.detect for a batch on the device (ctpn_text_lines).  rois [B,rows,5] float32 and count [B] int32:
        the proposal layer's output on this device (blob coordinates, rows in any order); im_hw [B,2] the (h, w) frame of
        the lines (resize_im's output size) and im_scales [B] the blob scales, on the host.  mode "H" (axis-aligned, clipped)
        or "O" (oriented); cfg: the 9 connector constants (see textlines.DEFAULT_CFG; None = those defaults).  Returns device
        tensors (lines [B,rows,9] float64, num [B] int32, status [B] int32) without synchronising; for each image the first
        num[b] rows equal textlines.text_lines(rois[b, :count[b], 1:5] / np.float64(im_scales[b]), rois[b, :count[b], 0],
        im_hw[b], mode, cfg) bit for bit, and status[b] != 0 where that call would raise (see split_lines).
        out=(lines, num, status): write into these contiguous tensors (e.g. views of a packed buffer, unpack_lines)."""
        if mode not in ("H", "O"):
            raise ValueError("mode must be 'H' or 'O' (got %r)" % (mode,))
        assert rois.is_cuda and rois.dtype == torch.float32 and rois.dim() == 3 and rois.shape[2] == 5
        assert count.is_cuda and count.dtype == torch.int32 and count.shape == (rois.shape[0],)
        B, rows = int(rois.shape[0]), int(rois.shape[1])
        hw = np.ascontiguousarray(np.asarray(im_hw, np.int64).reshape(-1, 2).astype(np.int32))
        sc = np.ascontiguousarray(np.asarray(im_scales, np.float64).reshape(-1))
        if hw.shape[0] != B or sc.shape[0] != B:
            raise ValueError("text_lines: %d images but %d sizes and %d scales" % (B, hw.shape[0], sc.shape[0]))
        cfg9 = None if cfg is None else np.ascontiguousarray(cfg, np.float32).reshape(9)
        need = N.lib.ctpn_text_lines_workspace_bytes(B, rows, max(1, int(hw[:, 1].max())))
        ws = self._workspace(ws_key, need)
        if out is not None:
            lines, num, status = out
            assert lines.shape == (B, rows, 9) and lines.dtype == torch.float64 and num.shape == status.shape == (B,)
            assert lines.is_contiguous() and num.is_contiguous() and status.is_contiguous()
        else:
            lines = torch.empty((B, rows, 9), dtype=torch.float64, device=self.device)
            num = torch.empty((B,), dtype=torch.int32, device=self.device)
            status = torch.empty((B,), dtype=torch.int32, device=self.device)
        N.check(N.lib.ctpn_text_lines(N.ptr(rois.contiguous()), N.ptr(count.contiguous()), B, rows, N.ptr(hw), N.ptr(sc), 1 if mode == "O" else 0,
                                      N.ptr(cfg9), N.ptr(lines), N.ptr(num), N.ptr(status), N.ptr(ws), ws.numel(), N.stream_ptr()),
                "ctpn_text_lines")
        return lines, num, status

    @staticmethod
    def split_lines(lines, num, status, im_hw=None):
        """Host copies of text_lines' results -> one float64 [num[b], 9] array per image.  Raises CtpnError for an image
        whose status is nonzero, as the host connector raises on it (status 1: a proposal's x1 outside the image width,
        where the reference raises IndexError; 2: a count outside [0, rows])."""
        lines, num, status = (t.cpu().numpy() if torch.is_tensor(t) else np.asarray(t) for t in (lines, num, status))
        out = []
        for b in range(lines.shape[0]):
            st = int(status[b])
            if st == 1:
                width = "" if im_hw is None else " %d" % int(np.asarray(im_hw).reshape(-1, 2)[b, 1])
                raise N.CtpnError("text lines of image %d: a proposal's x1 lies outside the image width%s" % (b, width))
            if st:
                raise N.CtpnError("text lines of image %d: status %d (proposal count outside [0, rows])" % (b, st))
            out.append(lines[b, :int(num[b])].copy())
        return out

    def detect_lines_images(self, images, mode="H", resize=True, max_batch=32, return_resized=False, scale=600, max_scale=1200,
                            cfg=None, channels="BGR", crop_height=None, crop_from="resized"):
        """ctpn() (demo.py:55-68 minus file I/O) for a list of raw HxWx3 uint8 BGR images of any sizes, all on the device:
        the batches of rois_images (same inputs and batching), then the text-line connector (text_lines) on each batch's
        rois, and one D2H per batch of the packed lines, counts and statuses.  Returns, in input order, (lines float64
        [m,9] (x1,y1,x2,y2,x3,y3,x4,y4,score) in the resize_im frame, f) per image, plus the resize_im output with
        return_resized.  lines is bit-identical to TextDetector(native=True).detect(boxes, scores[:, None], resized.shape[:2])
        on detect_images' output for that image (mode "H" / "O" as cfg.TEST.DETECT_MODE; cfg: the 9 connector constants,
        None = text_connect_cfg's).  Raises CtpnError where that connector raises (a proposal outside the image width).
        images and channels: as for rois_images (host images, or CUDA tensors read in place; BGR or RGB).

        crop_height=Hc (2..256): each tuple becomes (lines, f, crops, widths) (plus resized): crops a CUDA uint8
        [m, Hc, max(widths), 3] tensor whose crops[j, :, :widths[j]] is line j cut out of the resize_im output as a line
        recognizer takes it -- cv2.warpAffine(resized, Minv, (widths[j], Hc), INTER_LINEAR | WARP_INVERSE_MAP,
        BORDER_REPLICATE) with the map of include/ctpn_b200.h (ctpn_line_crops_u8), bit for bit -- and zeros past
        widths[j]; widths an int64 array [m].  The crops are cut on the device from the canvas the lines were found on: no
        image byte comes back for them and nothing goes up.  They are ready on the stream that was current when the call
        was made.

        crop_from="source" (with crop_height): the crops are cut out of the source photo at full resolution instead of the
        resize_im canvas -- crops[j, :, :widths[j]] is the same recipe applied to the source line lines[j, :8] / f (float64,
        the division draw_boxes makes) and the source image in BGR: a host image as passed (flipped with channels="RGB"),
        a tensor read through its strides, a YUV420 frame as cv2.cvtColor converts it (ctpn_line_crops_strided_u8 /
        ctpn_line_crops_yuv420_u8).  The lines stay in the resize_im frame; widths are the source widths.  The sources are
        read where they already are on the device -- host images in the batch's upload, tensors and frames in place -- so
        nothing more crosses the bus.  With f = 1 (resize=False, or a photo already at `scale`) both settings give the
        same crops.  crop_from="resized" (default) is the canvas crop above."""
        if mode not in ("H", "O"):
            raise ValueError("mode must be 'H' or 'O' (got %r)" % (mode,))
        check_crop_height(crop_height, "detect_lines_images")
        check_crop_from(crop_from, crop_height, "detect_lines_images")
        rows = self.result_rows()
        stream = torch.cuda.current_stream()

        def connect(packed, items):
            return self._connect(packed, items, mode, cfg)

        out = [None] * len(images)
        for idxs, items, out_h, resized, u8, res, sources in self._images_batches(images, resize, max_batch, return_resized,
                                                                                  scale, max_scale, "detect_lines_images",
                                                                                  after=connect, channels=channels):
            per_image = self.split_lines(*self.unpack_lines(out_h.numpy(), len(idxs), rows), im_hw=[p.resized for p in items])
            crops = [()] * len(idxs)
            if crop_height is not None:     # before the next batch's front-end rewrites the canvas and sources, in stream order
                crops = self._line_crops(u8, res, items, per_image, crop_height, stream,
                                         sources() if crop_from == "source" else None)
            for k, (i, lines) in enumerate(zip(idxs, per_image)):
                out[i] = (lines, items[k].f) + crops[k] + ((resized[k],) if return_resized else ())
        return out

    def detect_images(self, images, resize=True, max_batch=32, return_resized=False, scale=600, max_scale=1200, channels="BGR"):
        """rois_images as test_ctpn returns it: per image (scores float32 [n], boxes float64 [n,4] = rois / im_scale, f), plus
        the resize_im output with return_resized.  Boxes are in the resize_im frame, as TextDetector expects them
        (draw_boxes divides by f).  images and channels: as for rois_images."""
        res = self.rois_images(images, resize=resize, max_batch=max_batch, return_resized=return_resized, scale=scale,
                               max_scale=max_scale, channels=channels)
        return [(r[0][:, 0], r[0][:, 1:5] / np.float64(r[1])) + tuple(r[2:]) for r in res]

    # ---- streamed photos: staging, upload and compute overlapped ---------------------------------
    def _stream_buffer(self, kind, slot, nbytes, stream=None):
        """Grow-only uint8 buffer `kind` of pipeline slot `slot`: pinned host memory for kind "pin_*", else device memory
        (allocated in `stream`'s pool).  A buffer is replaced only by a larger one (sizes are powers of two), after the
        device has finished with the old one."""
        bufs = self.__dict__.setdefault("_stream_buffers", {})
        buf = bufs.get((kind, slot))
        if buf is None or buf.numel() < nbytes:
            torch.cuda.synchronize(self.device)
            size = 1 << max(20, (int(nbytes) - 1).bit_length())
            if kind.startswith("pin_"):
                buf = torch.empty(size, dtype=torch.uint8, pin_memory=True)
            else:
                # see rois_batches: a buffer another stream writes must not be a block the compute stream's tensors
                # have just released, so it comes from that stream's pool
                with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream()):
                    buf = torch.empty(size, dtype=torch.uint8, device=self.device)
                torch.cuda.synchronize(self.device)
            bufs[(kind, slot)] = buf
        return buf

    def _stream(self, images, split, what, resize, max_batch, return_resized, scale, max_scale, window, compact_rows, after=None,
                channels="BGR", crop=None, source_crops=False):
        """The generator behind stream_rois_images / stream_images / stream_lines_images: run_stream over the batches of
        stream_windows with these stages, on two slots used alternately --
          pack     (worker thread) the batch's rows, row maps, sizes and im_info into the slot's pinned buffer
                   (stream_layout), once the upload that last read that buffer has finished;
          upload   one H2D of that buffer on the copy stream, once the compute that last read the slot's device buffer has
                   finished;
          compute  on the current stream: the front-end kernels, detect_packed and after(packed, items), as _images_batches
                   runs them, into the slot's uint8 canvas; then on the result stream one D2H of the result (and, with
                   return_resized, one of the uint8 canvas);
          finish   waits for that D2H and splits it: split(host buffer, batch) -> one tuple per image; then, with crop,
                   crop(tuples, batch, uint8 canvas, device result, compute stream, sources) -> the tuples extended, enqueued
                   on the compute stream before the next compute, which reuses the slot's canvas, is.
        source_crops (crop reads the sources, line_crop_sources): host images are uploaded whole (a line may lie on any
        row, so compact_rows does not apply), into a ring of three device buffers indexed by batch number: the crop of
        batch k - 1 is enqueued after upload(k + 1), so with two buffers that upload would overwrite its pixels; upload
        (k + 1) reuses the buffer of batch k - 2 once that batch's crop has run.  Tensors and frames are recorded on the
        compute stream after their crop, so their memory outlives it whatever the caller drops.
        The host blocks only in finish, for the batch it is about to yield.  A stream of CUDA tensors (its first image
        decides) packs and uploads the sizes and im_info only, and compute reads the tensors in place
        (ctpn_resize_linear_u8_strided); each batch holds its tensors until its results have come back."""
        if not 1 <= int(max_batch) <= 64:
            raise ValueError("%s: max_batch must be 1..64 (the ragged front-end kernels take up to 64 images)" % what)
        window = 2 * int(max_batch) if window is None else int(window)
        if window < 1:
            raise ValueError("%s: window must be at least 1" % what)
        check_channels(channels, what)
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
            self._result_stream = torch.cuda.Stream(device=self.device)
        copy_stream, result_stream = self._copy_stream, self._result_stream
        main = torch.cuda.current_stream()
        lut = self._mean_lut()
        copied, computed, returned = [None, None], [None, None], [None, None]     # per slot: events of its last H2D / compute / D2H
        cropped, uploads = [None] * 3, [0]     # source crops: per ring buffer, the event after the last crop that read it
        if source_crops:
            compact_rows = False

        device_images = []                      # [the kind (on_device) of the stream's images], set by its first image

        def prepare(im, index):
            dev = on_device(im, self.device, what, index, channels)
            if not device_images:
                device_images.append(dev)
            elif dev != device_images[0]:
                raise mixed_kinds(what, index, dev, device_images[0], "the stream's first image")
            a = im if dev else (im.numpy() if torch.is_tensor(im) else np.asarray(im))
            return a, frontend_plan([a], resize=resize, scale=scale, max_scale=max_scale, cfg=self.cfg, first=index)[0]

        def pack_on_host(batch, slot):          # calling thread: sizes only, and the pinned buffer (grow-only)
            lay = stream_layout(batch.items, [tuple(im.shape[:2]) for im in batch.images], compact_rows,
                                sources=not device_images[0])
            return lay, self._stream_buffer("pin_src", slot, lay.total), copied[slot]

        def pack(batch, slot, staged):          # worker thread: row copies (numpy releases the GIL for them)
            lay, pinned, free = staged
            if free is not None:
                free.synchronize()
            stream_pack(pinned.numpy(), lay, batch, channels)
            return lay, pinned

        def upload(batch, slot, packed):
            lay, pinned = packed
            ring = uploads[0] % 3 if source_crops else slot
            uploads[0] += 1
            free = cropped[ring] if source_crops else computed[slot]
            dev = self._stream_buffer("src", ring, lay.total, copy_stream)
            with torch.cuda.stream(copy_stream):
                if free is not None:
                    copy_stream.wait_event(free)
                dev[:lay.total].copy_(pinned[:lay.total], non_blocking=True)          # the batch's one H2D
                copied[slot] = torch.cuda.Event()
                copied[slot].record(copy_stream)
            return lay, dev, copied[slot], ring

        def compute(batch, slot, uploaded):
            lay, dev, arrived, ring = uploaded
            items, (H, W) = batch.items, batch.canvas
            B = len(items)
            stream = N.stream_ptr()
            main.wait_event(arrived)
            if returned[slot] is not None:
                main.wait_event(returned[slot])        # the D2H out of this slot's uint8 canvas
            is_u8 = items[0].dtype == "|u1"
            Hr, Wr = (H, W) if is_u8 else (max(p.resized[0] for p in items), max(p.resized[1] for p in items))
            u8 = self._stream_buffer("u8", slot, B * Hr * Wr * 3)[:B * Hr * Wr * 3].view(B, Hr, Wr, 3)
            fxy = np.array([[p.f, p.f] for p in items], np.float64)
            resized_hw = np.array([p.resized for p in items], np.int32)
            if lay.offsets is None:
                resize_in_place(batch.images, device_images[0], channels, fxy, resized_hw, u8, stream)
            elif lay.maps is None:
                hwp = np.array([im.shape[:2] + (im.shape[1],) for im in batch.images], np.int32)
                N.check(N.lib.ctpn_resize_linear_u8_ragged(N.ptr(dev), lay.map_base, N.ptr(lay.offsets), N.ptr(hwp), N.ptr(fxy),
                                                           N.ptr(resized_hw), B, 3, N.ptr(u8), Hr, Wr, stream),
                        "ctpn_resize_linear_u8_ragged")
            else:
                hwp = np.array([im.shape[:2] + (im.shape[1],) for im in batch.images], np.int32)
                maps = dev[lay.map_base:lay.sizes_at].view(torch.int32)
                N.check(N.lib.ctpn_resize_linear_u8_ragged_rows(N.ptr(dev), lay.map_base, N.ptr(lay.offsets), N.ptr(hwp),
                                                                N.ptr(lay.stored), N.ptr(maps), maps.numel(), N.ptr(lay.maps),
                                                                N.ptr(fxy), N.ptr(resized_hw), B, 3, N.ptr(u8), Hr, Wr, stream),
                        "ctpn_resize_linear_u8_ragged_rows")
            canvas = u8
            if not is_u8:
                canvas = self._workspace("stream_blob", B * H * W * 12)[:B * H * W * 12].view(torch.float32).view(B, H, W, 3)
                boffs = np.arange(B, dtype=np.int64) * (Hr * Wr * 3)
                bhwp = np.concatenate([resized_hw, np.full((B, 1), Wr, np.int32)], axis=1)
                bfxy = np.array([[p.im_scale, p.im_scale] for p in items], np.float64)
                blob_hw = np.array([p.blob for p in items], np.int32)
                N.check(N.lib.ctpn_image_blob_f32_ragged(N.ptr(u8), B * Hr * Wr * 3, N.ptr(boffs), N.ptr(bhwp), N.ptr(bfxy),
                                                         N.ptr(blob_hw), N.ptr(lut), B, N.ptr(canvas), H, W, stream),
                        "ctpn_image_blob_f32_ragged")
            tail = dev[lay.sizes_at:lay.total]
            ints = tail[:16 * B].view(torch.int32)
            packed = self.detect_packed(canvas, tail[16 * B:].view(torch.float32).view(B, 3), sizes=np.array([p.blob for p in items]),
                                        device_sizes=(ints[:2 * B].view(B, 2), ints[2 * B:].view(B, 2)))
            result = packed if after is None else after(packed, items)
            computed[slot] = torch.cuda.Event()
            computed[slot].record(main)
            nbytes = result.numel() * result.element_size()
            with torch.cuda.stream(result_stream):
                result_stream.wait_event(computed[slot])
                out_h = self._stream_buffer("pin_out", slot, nbytes)[:nbytes].view(result.dtype)
                out_h.copy_(result, non_blocking=True)                                  # one D2H: the packed results
                res_h = None
                if return_resized:                                                      # and one for the resize_im outputs
                    res_h = self._stream_buffer("pin_u8", slot, u8.numel())[:u8.numel()].view(B, Hr, Wr, 3)
                    res_h.copy_(u8, non_blocking=True)
                returned[slot] = torch.cuda.Event()
                returned[slot].record(result_stream)
            # the device results and the batch's input tensors live until the D2H, which follows the compute, has run
            return out_h, res_h, returned[slot], (packed, result, batch.images, u8, lay, dev, ring)

        def finish(batch, handle):
            out_h, res_h, ev, keep = handle
            ev.synchronize()
            per_image = split(out_h, batch)
            if crop is not None:
                lay, dev, ring = keep[4:]
                sources = None
                if source_crops:
                    sources = line_crop_sources(batch.images, device_images[0], channels, dev, lay.offsets)
                per_image = crop(per_image, batch, keep[3], keep[1], main, sources)
                if source_crops:
                    cropped[ring] = torch.cuda.Event()
                    cropped[ring].record(main)
                    for t in batch.images if device_images[0] else ():
                        for p in (t if device_images[0] == FRAME else (t,)):
                            p.record_stream(main)
            if res_h is not None:
                rn = res_h.numpy()
                per_image = [t + (rn[k, :p.resized[0], :p.resized[1]].copy(),) for k, (t, p) in enumerate(zip(per_image, batch.items))]
            return per_image

        def drain():
            for st in (copy_stream, main, result_stream):
                st.synchronize()
            self._streaming = False

        def stream():
            if getattr(self, "_streaming", False):
                raise RuntimeError("%s: another stream of this engine is still open (its slots are in use); close it first" % what)
            self._streaming = True
            yield from run_stream(stream_windows(images, window, max_batch, prepare), pack_on_host, pack, upload, compute, finish,
                                  drain)

        return stream()

    def stream_rois_images(self, images, resize=True, max_batch=32, return_resized=False, scale=600, max_scale=1200, window=None,
                           compact_rows=True, channels="BGR"):
        """rois_images for any iterable of raw HxWx3 uint8 BGR images (e.g. a generator that decodes files), as a generator:
        yields, in input order, the tuple rois_images returns for each image -- bit-identical to it -- while later images
        are still being pulled, packed, uploaded and computed (see _stream for the stages that overlap).  window: how
        many images are pulled from the iterable before their ragged batches are planned (default 2 * max_batch); it
        bounds the memory held and, like max_batch, changes which images share a batch, never a result.  A camera-size
        photo is uploaded as the rows resize_im reads only (FrontendStep.rows; compact_rows=False uploads every image
        whole).  A bad image raises frontend_plan's ValueError when the stream reaches it, after the results of all images
        before it.  Closing the generator early waits for the work in flight and leaves the engine ready for any other
        call; one stream per engine can be open at a time.

        The images may instead all be CUDA uint8 [H, W, 3] tensors on this engine's device, at any strides, as rois_images
        takes them: then only the sizes and im_info are uploaded, and the kernels read the tensors in place.  They must be
        ready on the stream that was current when the generator was created (torch's rule); the engine synchronises
        nothing for them.  The stream keeps each batch's tensors referenced until that batch's results have come back, so
        a caller may drop its own references as soon as the generator has pulled them; the window then also bounds the
        device memory the stream holds.  YUV420 frames stream the same way (see rois_images), their planes held as tensors
        are.  An image of another kind than the stream's first (host image, CUDA tensor or YUV420 frame) raises ValueError
        when the stream reaches it, like a bad image.  channels: as for rois_images."""
        rows = self.result_rows()

        def split(out_h, batch):
            return [(r, p.im_scale, p.f) for r, p in zip(self._split_results(out_h, len(batch.items), rows), batch.items)]

        return self._stream(images, split, "stream_rois_images", resize, max_batch, return_resized, scale, max_scale, window,
                            compact_rows, channels=channels)

    def stream_images(self, images, resize=True, max_batch=32, return_resized=False, scale=600, max_scale=1200, window=None,
                      compact_rows=True, channels="BGR"):
        """detect_images as a generator over any iterable of raw photos: see stream_rois_images."""
        rows = self.result_rows()

        def split(out_h, batch):
            return [(r[:, 0], r[:, 1:5] / np.float64(p.im_scale), p.f)
                    for r, p in zip(self._split_results(out_h, len(batch.items), rows), batch.items)]

        return self._stream(images, split, "stream_images", resize, max_batch, return_resized, scale, max_scale, window,
                            compact_rows, channels=channels)

    def stream_lines_images(self, images, mode="H", resize=True, max_batch=32, return_resized=False, scale=600, max_scale=1200,
                            cfg=None, window=None, compact_rows=True, channels="BGR", crop_height=None, crop_from="resized"):
        """detect_lines_images as a generator over any iterable of raw photos: see stream_rois_images; the connector runs
        on each batch's rois on the device and only the lines come back.  Raises CtpnError where detect_lines_images does.
        crop_height: as for detect_lines_images; a batch's crops are cut when its lines have come back, before the canvas
        is reused, on the stream that was current when the generator was created, and stay valid after it is closed.
        crop_from="source": as for detect_lines_images.  Host photos are then uploaded whole, whatever compact_rows says
        (a line may lie on any source row, and its rows are known only once the lines are back), and the stream reads
        tensors and frames until their crops have run, which are enqueued before their results are yielded."""
        if mode not in ("H", "O"):
            raise ValueError("mode must be 'H' or 'O' (got %r)" % (mode,))
        check_crop_height(crop_height, "stream_lines_images")
        check_crop_from(crop_from, crop_height, "stream_lines_images")
        rows = self.result_rows()

        def split(out_h, batch):
            hw = [p.resized for p in batch.items]
            lines = self.split_lines(*self.unpack_lines(out_h.numpy(), len(hw), rows), im_hw=hw)
            return [(ln, p.f) for ln, p in zip(lines, batch.items)]

        crop = None
        if crop_height is not None:
            def crop(per_image, batch, u8, res, stream, sources):
                crops = self._line_crops(u8, res, batch.items, [t[0] for t in per_image], crop_height, stream, sources)
                return [t + c for t, c in zip(per_image, crops)]

        return self._stream(images, split, "stream_lines_images", resize, max_batch, return_resized, scale, max_scale, window,
                            compact_rows, after=lambda packed, items: self._connect(packed, items, mode, cfg), channels=channels,
                            crop=crop, source_crops=crop_from == "source")

    def _connect(self, packed, items, mode, cfg):
        """The text-line connector on one batch's packed rois -> the packed lines (unpack_lines), on the device."""
        B, rows = len(items), self.result_rows()
        rois, count = self.unpack(packed, B, rows)
        res = torch.empty(B * rows * 9 + B, dtype=torch.float64, device=self.device)
        self.text_lines(rois, count, [p.resized for p in items], [p.im_scale for p in items], mode, cfg,
                        out=self.unpack_lines(res, B, rows))
        return res

    def _line_crops(self, u8, res, items, lines, crop_height, stream, sources=None):
        """The line crops of one batch on `stream` (ctpn_line_crops_u8): u8 the batch's uint8 resize_im canvas [B, Hr, Wr, 3],
        res its packed device lines (_connect), lines the same lines on the host, one float64 [m, 9] array per image.
        sources (line_crop_sources): cut from the batch's source images instead (ctpn_line_crops_strided_u8 /
        ctpn_line_crops_yuv420_u8), at the source widths -- of lines / f, divided here as the kernel divides them.
        Returns one (crops, widths) pair per image.  Each image's widths are computed on the host
        (ctpn_line_crop_widths_host) and travel with the launch by value, with the output pointers.  The kernel recomputes
        every width from the device lines; one that differs sets the image's entry of the engine's status array, which
        this method checks at each call -- so such a fault, which one shared width definition rules out, is raised by the
        next crop call that finds it."""
        B, rows, hc = len(items), self.result_rows(), int(crop_height)
        status = self._crop_status_buffer()
        widths, crops = [], []
        with torch.cuda.stream(stream):
            for b, ln in enumerate(lines):
                ln = np.array(ln, np.float64)
                if sources is not None:
                    ln[:, :8] /= np.float64(items[b].f)
                w = np.zeros(len(ln), np.int32)
                N.check(N.lib.ctpn_line_crop_widths_host(N.ptr(ln), len(ln), hc, N.ptr(w)),
                        "ctpn_line_crop_widths_host (image %d of the batch)" % b)
                widths.append(w.astype(np.int64))
                crops.append(torch.empty((len(ln), hc, int(w.max()) if len(w) else 0, 3), dtype=torch.uint8,
                                         device=self.device))
            hw = np.array([p.resized for p in items], np.int32)
            num = np.array([len(w) for w in widths], np.int32)
            wmax = np.array([int(w.max()) if len(w) else 0 for w in widths], np.int32)
            outs = np.array([c.data_ptr() for c in crops], np.uint64)
            if sources is None:
                Hr, Wr = int(u8.shape[1]), int(u8.shape[2])
                N.check(N.lib.ctpn_line_crops_u8(N.ptr(u8), Hr * Wr * 3, Wr * 3, N.ptr(hw), N.ptr(res), B, rows, hc,
                                                 N.ptr(num), N.ptr(wmax), N.ptr(outs), N.ptr(status), N.stream_ptr(stream)),
                        "ctpn_line_crops_u8")
            else:
                yuv, desc, src_hw = sources
                name = "ctpn_line_crops_yuv420_u8" if yuv else "ctpn_line_crops_strided_u8"
                addr, nbytes, offs, strides = descriptor_arrays(desc)
                f = np.array([p.f for p in items], np.float64)
                N.check(getattr(N.lib, name)(N.ptr(addr), N.ptr(nbytes), N.ptr(offs), N.ptr(strides), N.ptr(src_hw), N.ptr(f),
                                             N.ptr(res), B, rows, hc, N.ptr(num), N.ptr(wmax), N.ptr(outs), N.ptr(status),
                                             N.stream_ptr(stream)), name)
        return [(c, w) for c, w in zip(crops, widths)]

    def _crop_status_buffer(self):
        """The engine's pinned int32 [64] crop status array, which the crop kernel writes through the unified address space
        (no copy); raises CtpnError, and clears it, when an earlier launch has set an entry."""
        st = getattr(self, "_crop_status", None)
        if st is None:
            st = self._crop_status = torch.zeros(64, dtype=torch.int32, pin_memory=True)
        if bool(st.any()):
            st.zero_()
            raise N.CtpnError("ctpn_line_crops_u8: a line's crop width on the device differed from the host's; its crop was "
                              "not written")
        return st

    def detect(self, image, im_scale=1.0):
        """Single image [H,W,3] -> (scores, boxes); the test_ctpn() contract."""
        return self.detect_batch(image[None], im_scale)[0]


def ragged_plan(shapes, dtypes, max_batch=32):
    """Batches of a ragged detect (Engine.detect_ragged): shapes [(H, W)], dtypes [str] of n images -> a list of
    (indices, (canvas_H, canvas_W)).  Images are grouped by dtype and orientation (H > W or not), sorted by (H, W) within a
    group, and each group is cut into chunks of at most max_batch; a chunk's canvas is its largest H and largest W.  Every
    index appears in exactly one chunk."""
    max_batch = int(max_batch)
    if max_batch < 1:
        raise ValueError("ragged_plan: max_batch must be >= 1")
    if len(shapes) != len(dtypes):
        raise ValueError("ragged_plan: %d shapes but %d dtypes" % (len(shapes), len(dtypes)))
    groups = {}
    for i, ((h, w), dt) in enumerate(zip(shapes, dtypes)):
        groups.setdefault((str(dt), int(h) > int(w)), []).append(i)
    plan = []
    for key in sorted(groups):
        idxs = sorted(groups[key], key=lambda i: (int(shapes[i][0]), int(shapes[i][1]), i))
        for k in range(0, len(idxs), max_batch):
            part = idxs[k:k + max_batch]
            plan.append((part, (max(int(shapes[i][0]) for i in part), max(int(shapes[i][1]) for i in part))))
    return plan


FrontendStep = collections.namedtuple("FrontendStep", "f resized im_scale blob dtype rows", defaults=(None,))


def frontend_rows(h, f_y, out_h):
    """The source rows that resize_im's cv2.resize of an h-row uint8 image by f_y to out_h rows reads: sorted, unique,
    int64.  INTER_LINEAR takes output row d from rows s and s + 1, s = floor(float32((d + 0.5) * (1 / f_y) - 0.5)), both
    clamped to [0, h - 1]; an exact 1/2 is routed to INTER_AREA, which reads every row."""
    h, out_h = int(h), int(out_h)
    scale = 1.0 / float(f_y)
    if scale == 2.0:
        return np.arange(h, dtype=np.int64)
    s = np.floor(((np.arange(out_h, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)).astype(np.int64)
    return np.unique(np.clip(np.concatenate([s, s + 1]), 0, h - 1))


def _cv_round_size(h, w, s):
    return int(np.rint(float(h) * s)), int(np.rint(float(w) * s))        # cvRound: round half to even, in float64


def frontend_plan(shapes, resize=True, scale=600, max_scale=1200, cfg=None, first=0):
    """What the demo's host front-end does to each image, computed on the host: shapes is a list of HxWx3 uint8 images
    (anything with .shape and .dtype) or of (H, W[, 3]) tuples.  Per image a FrontendStep of
      f         the resize_im factor (ctpn/demo.py: short side -> scale unless the long side would exceed max_scale;
                1.0 with resize=False, for images already at that scale),
      resized   its (h, w) as cv2.resize computes it (cvRound),
      im_scale  _get_image_blob's scale (lib/fast_rcnn/test.py _im_scale: SCALES[0] / short side, or MAX_SIZE / long side
                when np.round(im_scale * long side) > MAX_SIZE; cfg: SCALES and MAX_SIZE, default DEFAULT_CFG),
      blob      the (h, w) of the blob the network sees,
      dtype     '|u1' when im_scale == 1 (the uint8 image is the blob), else '<f4' (the float32 rescale),
      rows      the source rows resize_im reads (frontend_rows, as a tuple) when they are at most 3/4 of the image -- a
                streamed upload then sends only those (Engine.stream_rois_images) -- or None: send the image densely.
    Error messages number the images from `first` (a stream plans its images one at a time).  Raises ValueError when an image is not HxWx3 uint8, a resize would be empty or a blob side would be under 16.
    A YUV420 frame plans as the BGR image it converts to; one with odd sides or malformed planes raises ValueError."""
    c = dict(DEFAULT_CFG)
    if cfg:
        c.update(cfg)
    target, max_size = float(c["SCALES"][0]), float(c["MAX_SIZE"])
    out = []
    for i, s in enumerate(shapes, int(first)):
        if isinstance(s, YUV420):
            s = s.hw("frontend_plan", i)
        elif hasattr(s, "shape") and hasattr(s, "dtype"):
            if len(s.shape) != 3 or s.shape[2] != 3 or str(s.dtype) not in ("uint8", "torch.uint8"):
                raise ValueError("frontend_plan: image %d must be HxWx3 uint8 (got %s %s)" % (i, tuple(s.shape), s.dtype))
            s = tuple(s.shape)
        s = tuple(int(v) for v in s)
        if len(s) not in (2, 3) or (len(s) == 3 and s[2] != 3):
            raise ValueError("frontend_plan: image %d must be HxWx3 uint8 (got shape %s)" % (i, s))
        h, w = s[:2]
        if h < 1 or w < 1:
            raise ValueError("frontend_plan: image %d is empty (%dx%d)" % (i, h, w))
        f = 1.0
        if resize:
            f = float(scale) / min(h, w)
            if max_scale is not None and f * max(h, w) > max_scale:
                f = float(max_scale) / max(h, w)
        rh, rw = _cv_round_size(h, w, f)
        if rh < 1 or rw < 1:
            raise ValueError("frontend_plan: image %d (%dx%d) resizes to nothing at f = %r" % (i, h, w, f))
        im_scale = target / float(min(rh, rw))
        if np.round(im_scale * max(rh, rw)) > max_size:
            im_scale = max_size / float(max(rh, rw))
        bh, bw = (rh, rw) if im_scale == 1.0 else _cv_round_size(rh, rw, im_scale)
        if bh < 16 or bw < 16:
            raise ValueError("frontend_plan: image %d (%dx%d) gives a %dx%d blob; both sides must be at least 16" % (i, h, w, bh, bw))
        rows = None
        if f < 0.5:            # at 1/2 and above the two taps of consecutive output rows cover every source row
            live = frontend_rows(h, f, rh)
            if 4 * len(live) <= 3 * h:
                rows = tuple(int(r) for r in live)
        out.append(FrontendStep(f, (rh, rw), im_scale, (bh, bw), "|u1" if im_scale == 1.0 else "<f4", rows))
    return out


# ---- photos already in device memory ------------------------------------------------------------------------------------
CHANNELS = ("BGR", "RGB")


def check_crop_height(crop_height, what):
    """crop_height of the line calls: None (no crops) or an int 2..256."""
    if crop_height is None:
        return
    if isinstance(crop_height, (bool, np.bool_)) or not isinstance(crop_height, (int, np.integer)) or not 2 <= crop_height <= 256:
        raise ValueError("%s: crop_height must be None or an int 2..256 (got %r)" % (what, crop_height))


CROP_FROM = ("resized", "source")


def check_crop_from(crop_from, crop_height, what):
    """crop_from of the line calls: "resized" (crops out of the resize_im canvas) or "source" (out of the source images),
    the latter only with a crop_height."""
    if not isinstance(crop_from, str) or crop_from not in CROP_FROM:
        raise ValueError("%s: crop_from must be 'resized' or 'source' (got %r)" % (what, crop_from))
    if crop_from == "source" and crop_height is None:
        raise ValueError("%s: crop_from='source' needs a crop_height" % what)


def check_channels(channels, what):
    if channels not in CHANNELS:
        raise ValueError("%s: channels must be 'BGR' or 'RGB' (got %r)" % (what, channels))


def as_bgr(a, channels):
    """A host image as the BGR view the packing copy reads (no copy of its own)."""
    return a[:, :, ::-1] if channels == "RGB" else a


class YUV420(collections.namedtuple("YUV420", "y u v")):
    """A YUV 4:2:0 video frame in device memory, as the raw-photo calls of Engine take it: y a uint8 [H, W] tensor, u and
    v uint8 [H/2, W/2] tensors, H and W even, at any strides (views into one buffer, or separate allocations).  The calls
    convert it to BGR as cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / _NV21 / _I420 / _YV12) does -- BT.601 limited range,
    nearest chroma -- inside the resize (ctpn_resize_linear_u8_yuv420), and return what they return on that BGR image.
    That is cv2.cvtColor's conversion, not the one behind cv2.VideoCapture's BGR frames (FFmpeg's swscale rounds
    differently).  shape is that of the BGR image, (H, W, 3)."""
    __slots__ = ()
    LAYOUTS = ("NV12", "NV21", "I420", "YV12")

    @property
    def shape(self):
        return tuple(int(s) for s in self.y.shape[:2]) + (3,)

    @classmethod
    def from_buffer(cls, t, layout):
        """Views of the planes of one uint8 [H*3/2, W] buffer in cv2's layout `layout`: NV12 / NV21 -- H luma rows, then H/2
        rows of interleaved chroma (U first for NV12, V first for NV21); I420 / YV12 -- H luma rows, then the U and V
        planes (V first for YV12) with two chroma rows per buffer row.  The rows may be pitched (any row stride); an I420 /
        YV12 buffer then has its chroma rows at half the luma pitch, and must have a column stride of 1 and an even row
        stride.  Raises ValueError on what cannot be viewed so."""
        if layout not in cls.LAYOUTS:
            raise ValueError("YUV420.from_buffer: layout must be one of %s (got %r)" % ("/".join(cls.LAYOUTS), layout))
        if not torch.is_tensor(t) or t.dtype != torch.uint8 or t.dim() != 2:
            raise ValueError("YUV420.from_buffer: the buffer must be a uint8 [H*3/2, W] tensor")
        rows, W = int(t.shape[0]), int(t.shape[1])
        if rows % 3 or rows == 0 or W % 2 or W == 0:
            raise ValueError("YUV420.from_buffer: a %dx%d buffer is not [H*3/2, W] with H, W even and positive" % (rows, W))
        H = rows // 3 * 2
        y = t[:H]
        if layout in ("NV12", "NV21"):
            a, b = t[H:, 0::2], t[H:, 1::2]
            return cls(y, a, b) if layout == "NV12" else cls(y, b, a)
        pitch, col = t.stride()
        if col != 1 or pitch % 2 or pitch < W:
            raise ValueError("YUV420.from_buffer: an %s buffer needs rows of contiguous bytes at an even pitch >= W (got "
                             "strides %s)" % (layout, t.stride()))
        first = t.storage_offset() + H * pitch
        a = torch.as_strided(t, (H // 2, W // 2), (pitch // 2, 1), first)
        b = torch.as_strided(t, (H // 2, W // 2), (pitch // 2, 1), first + H // 2 * (pitch // 2))
        return cls(y, a, b) if layout == "I420" else cls(y, b, a)

    @classmethod
    def nv12(cls, y, uv):
        """A frame from a luma tensor y [H, W] and an interleaved U, V chroma tensor uv, [H/2, W] or [H/2, W/2, 2], which
        need not be adjacent to y (NVDEC surfaces).  Views, never copies."""
        if not torch.is_tensor(uv) or uv.dim() not in (2, 3) or (uv.dim() == 3 and uv.shape[2] != 2):
            raise ValueError("YUV420.nv12: uv must be a [H/2, W] or [H/2, W/2, 2] tensor")
        if uv.dim() == 3:
            return cls(y, uv[:, :, 0], uv[:, :, 1])
        return cls(y, uv[:, 0::2], uv[:, 1::2])

    def hw(self, what, index):
        """(H, W) of a well-formed frame; ValueError naming image `index` otherwise."""
        for name, p in zip("yuv", self):
            if not torch.is_tensor(p) or p.dtype != torch.uint8 or p.dim() != 2:
                raise ValueError("%s: image %d: YUV420 plane %s must be a 2-D uint8 tensor" % (what, index, name))
        H, W = (int(s) for s in self.y.shape)
        if H < 2 or W < 2 or H % 2 or W % 2:
            raise ValueError("%s: image %d is a %dx%d YUV420 frame; 4:2:0 frames have even sides" % (what, index, H, W))
        for name, p in zip("uv", self[1:]):
            if tuple(p.shape) != (H // 2, W // 2):
                raise ValueError("%s: image %d: YUV420 plane %s is %s, must be [%d, %d] for a %dx%d frame"
                                 % (what, index, name, tuple(p.shape), H // 2, W // 2, H, W))
        return H, W


# What the images of a raw-photo call are (on_device): host arrays, CUDA BGR / RGB tensors or YUV420 frames.  One call or
# stream takes one kind.  False / True keep on_device a truth value: whether the images are in device memory.
HOST, TENSOR, FRAME = False, True, "YUV420"
KIND_NAMES = {HOST: "a host image", TENSOR: "a CUDA tensor", FRAME: "a YUV420 frame"}


def on_device(im, device, what, index, channels="BGR"):
    """The kind of image `index` of a raw-photo call: HOST, TENSOR (a CUDA tensor) or FRAME (a YUV420 frame); a tensor or
    every plane of a frame must be on the engine's `device`, and a frame converts to BGR, so channels must be "BGR" (dtype
    and shape are frontend_plan's to check).  Anything else is a host image, CPU tensors included."""
    if isinstance(im, YUV420):
        for name, p in zip("yuv", im):
            if not (torch.is_tensor(p) and p.is_cuda):
                raise ValueError("%s: image %d: YUV420 plane %s is not a CUDA tensor; frames must be in device memory"
                                 % (what, index, name))
            if p.device != device:
                raise ValueError("%s: image %d: YUV420 plane %s is on %s, the engine runs on %s" % (what, index, name, p.device,
                                                                                                 device))
        if channels != "BGR":
            raise ValueError("%s: image %d is a YUV420 frame, which converts to BGR; channels=%r does not apply"
                             % (what, index, channels))
        return FRAME
    if not (torch.is_tensor(im) and im.is_cuda):
        return HOST
    if im.device != device:
        raise ValueError("%s: image %d is on %s, the engine runs on %s" % (what, index, im.device, device))
    return TENSOR


def mixed_kinds(what, index, kind, other, whose):
    return ValueError("%s: image %d is %s but %s is %s; a call or stream takes one kind (host images, CUDA tensors or YUV420 "
                      "frames), not both" % (what, index, KIND_NAMES[kind], whose, KIND_NAMES[other]))


def images_on_device(images, device, what, channels="BGR"):
    """The kind (on_device) of every image of a list call: HOST (False) when none is in device memory, TENSOR (True) or
    FRAME; a list of more than one kind raises ValueError."""
    kinds = [on_device(im, device, what, i, channels) for i, im in enumerate(images)]
    for i, k in enumerate(kinds):
        if k != kinds[0]:
            raise mixed_kinds(what, i, k, kinds[0], "image 0")
    return kinds[0] if kinds else HOST


def strided_descriptor(address, nbytes, offset, strides, channels="BGR"):
    """ctpn_resize_linear_u8_strided's descriptor of an HxWx3 uint8 image in the allocation at device `address` of `nbytes`
    bytes, whose sample (0, 0, 0) lies at byte `offset` and whose byte strides are strides = (row, column, channel) ->
    (address, nbytes, offset, (row, column, channel)) reading it as BGR.  channels="RGB": the image holds RGB, so the kernel
    starts at channel 2 and steps backwards."""
    check_channels(channels, "strided_descriptor")
    rs, cs, ks = (int(s) for s in strides)
    offset = int(offset)
    if channels == "RGB":
        offset, ks = offset + 2 * ks, -ks
    return int(address), int(nbytes), offset, (rs, cs, ks)


def tensor_descriptor(t, channels="BGR"):
    """strided_descriptor of a uint8 [H, W, 3] tensor: its storage is the allocation (uint8, so elements are bytes)."""
    st = t.untyped_storage()
    return strided_descriptor(st.data_ptr(), st.nbytes(), t.storage_offset(), t.stride(), channels)


def descriptor_arrays(desc):
    """The host arrays (addresses, bytes, offsets, strides) of a list of strided_descriptor / yuv420_descriptor tuples."""
    return (np.array([d[0] for d in desc], np.uint64), np.array([d[1] for d in desc], np.uint64),
            np.array([d[2] for d in desc], np.int64), np.array([d[3] for d in desc], np.int64))


def resize_strided(tensors, channels, fxy, dst_hw, dst, stream):
    """resize_im of CUDA uint8 [h, w, 3] tensors read in place into the uint8 canvas dst [B, H, W, 3]
    (ctpn_resize_linear_u8_strided)."""
    B = len(tensors)
    addr, nbytes, offs, strides = descriptor_arrays([tensor_descriptor(t, channels) for t in tensors])
    hw = np.array([tuple(t.shape[:2]) for t in tensors], np.int32)
    N.check(N.lib.ctpn_resize_linear_u8_strided(N.ptr(addr), N.ptr(nbytes), N.ptr(offs), N.ptr(strides), N.ptr(hw),
                                                N.ptr(np.ascontiguousarray(fxy, np.float64)),
                                                N.ptr(np.ascontiguousarray(dst_hw, np.int32)), B, N.ptr(dst),
                                                int(dst.shape[1]), int(dst.shape[2]), stream), "ctpn_resize_linear_u8_strided")


def yuv420_descriptor(frame):
    """ctpn_resize_linear_u8_yuv420's descriptor of a YUV420 frame: per plane (Y, U, V) (allocation address, its bytes,
    byte offset of sample (0, 0), (row, column) byte strides), from the planes' storages (uint8: elements are bytes)."""
    out = []
    for p in frame:
        st = p.untyped_storage()
        out.append((st.data_ptr(), st.nbytes(), p.storage_offset(), tuple(int(s) for s in p.stride())))
    return out


def resize_yuv420(frames, fxy, dst_hw, dst, stream):
    """resize_im of YUV420 frames, converted as cv2.cvtColor converts them, into the uint8 canvas dst [B, H, W, 3]
    (ctpn_resize_linear_u8_yuv420)."""
    B = len(frames)
    addr, nbytes, offs, strides = descriptor_arrays([d for f in frames for d in yuv420_descriptor(f)])
    hw = np.array([f.shape[:2] for f in frames], np.int32)
    N.check(N.lib.ctpn_resize_linear_u8_yuv420(N.ptr(addr), N.ptr(nbytes), N.ptr(offs), N.ptr(strides), N.ptr(hw),
                                               N.ptr(np.ascontiguousarray(fxy, np.float64)),
                                               N.ptr(np.ascontiguousarray(dst_hw, np.int32)), B, N.ptr(dst),
                                               int(dst.shape[1]), int(dst.shape[2]), stream), "ctpn_resize_linear_u8_yuv420")


def resize_in_place(images, kind, channels, fxy, dst_hw, dst, stream):
    """resize_im of images in device memory of one kind (on_device: TENSOR or FRAME), read in place, into dst."""
    if kind == FRAME:
        resize_yuv420(images, fxy, dst_hw, dst, stream)
    else:
        resize_strided(images, channels, fxy, dst_hw, dst, stream)


def line_crop_sources(images, kind, channels, buf=None, offsets=None):
    """The sources of a batch's source crops: (is YUV, descriptors, int32 [B, 2] source sizes) for
    ctpn_line_crops_strided_u8 / ctpn_line_crops_yuv420_u8.  Tensors and frames (kind TENSOR / FRAME) are read in place;
    host images (HOST) are read where their upload put them: whole, BGR, each at byte offsets[b] of the device buffer buf."""
    hw = np.array([tuple(im.shape[:2]) for im in images], np.int32).reshape(-1, 2)
    if kind == FRAME:
        return True, [d for f in images for d in yuv420_descriptor(f)], hw
    if kind == HOST:
        return False, [strided_descriptor(buf.data_ptr(), buf.numel(), int(o), (int(w) * 3, 3, 1))
                       for o, (h, w) in zip(offsets, hw)], hw
    return False, [tensor_descriptor(t, channels) for t in images], hw


# ---- streamed photos: the parts of Engine._stream that need no device ---------------------------------------------------
StreamBatch = collections.namedtuple("StreamBatch", "idxs items images canvas")
# One batch's upload: [the images' rows, back to back][row maps, int32][blob sizes, int32 B x 2][feature sizes, int32 B x 2]
# [im_info, float32 B x 3].  offsets / stored: per image, where its rows start (bytes) and how many it sends; rows: which
# (None: all); map_base: where the sources end and the maps start (a multiple of 4); maps: per image, where its map starts
# (int32 elements from map_base), or None when no image of the batch is compacted and there are no maps; sizes_at, total.
StreamLayout = collections.namedtuple("StreamLayout", "offsets stored rows map_base maps sizes_at total")


def stream_layout(items, shapes, compact_rows=True, sources=True):
    """Where everything of one batch goes in its upload buffer: items are the batch's FrontendSteps, shapes its images'
    (h, w).  An image is sent as its FrontendStep.rows when it has them (and compact_rows), else whole; if any image of the
    batch is compacted, every image gets a row map (the identity for a whole one).  sources=False (images the device reads
    in place): the buffer holds the sizes and im_info only."""
    if not sources:
        return StreamLayout(None, None, None, 0, None, 0, 28 * len(items))
    rows = [p.rows if compact_rows else None for p in items]
    stored = np.array([h if r is None else len(r) for (h, w), r in zip(shapes, rows)], np.int32)
    nbytes = [int(n) * int(w) * 3 for n, (h, w) in zip(stored, shapes)]
    offsets = np.cumsum([0] + nbytes[:-1]).astype(np.int64)
    map_base = (int(sum(nbytes)) + 3) & ~3
    maps, sizes_at = None, map_base
    if any(r is not None for r in rows):
        heights = [int(h) for h, w in shapes]
        maps = np.cumsum([0] + heights[:-1]).astype(np.int64)
        sizes_at += 4 * sum(heights)
    return StreamLayout(offsets, stored, rows, map_base, maps, sizes_at, sizes_at + 28 * len(items))


def stream_pack(buf, lay, batch, channels="BGR"):
    """Fills a batch's upload buffer (uint8 ndarray of at least lay.total bytes) as stream_layout laid it out; RGB images
    (channels="RGB") are flipped to BGR by the row copies."""
    B = len(batch.items)
    for k, im in enumerate(batch.images if lay.offsets is not None else ()):
        h, w = im.shape[:2]
        n, r = int(lay.stored[k]), lay.rows[k]
        dst = as_bgr(buf[lay.offsets[k]:lay.offsets[k] + n * w * 3].reshape(n, w, 3), channels)
        if r is None:
            dst[...] = im
        else:
            np.take(im, r, axis=0, out=dst, mode="clip")
        if lay.maps is not None:          # original row -> stored row; rows that are not stored are never looked up
            m = buf[lay.map_base + 4 * lay.maps[k]:lay.map_base + 4 * (lay.maps[k] + h)].view(np.int32)
            if r is None:
                m[:] = np.arange(h, dtype=np.int32)
            else:
                m[:] = 0
                m[np.asarray(r)] = np.arange(n, dtype=np.int32)
    blobs = np.array([p.blob for p in batch.items], np.int32)
    tail = buf[lay.sizes_at:lay.total]
    tail[:8 * B].view(np.int32)[:] = blobs.ravel()
    tail[8 * B:16 * B].view(np.int32)[:] = (blobs >> 4).ravel()
    tail[16 * B:].view(np.float32)[:] = np.array([[p.blob[0], p.blob[1], p.im_scale] for p in batch.items], np.float32).ravel()


def stream_windows(images, window, max_batch, prepare):
    """The ragged batches of a stream of images: pulls up to `window` images from the iterable, prepare(image, index) ->
    (array, FrontendStep) for each, plans them (ragged_plan) and yields their StreamBatches (idxs: positions in the stream);
    then the next window.  A ValueError of prepare is raised after the batches of the images before that image."""
    it = iter(images)
    first = 0
    while True:
        arrays, steps, bad = [], [], None
        for im in it:
            try:
                a, p = prepare(im, first + len(arrays))
            except ValueError as e:
                bad = e
                break
            arrays.append(a)
            steps.append(p)
            if len(arrays) == window:
                break
        for idxs, canvas in ragged_plan([p.blob for p in steps], [p.dtype for p in steps], max_batch):
            yield StreamBatch([first + i for i in idxs], [steps[i] for i in idxs], [arrays[i] for i in idxs], canvas)
        if bad is not None:
            raise bad
        if len(arrays) < window:
            return
        first += len(arrays)


def run_stream(batches, stage, pack, upload, compute, finish, drain):
    """Drives a stream of StreamBatches through a two-slot pipeline and yields every image's result in stream order.
    Batch k uses slot k & 1.  stage(batch, slot) runs on the calling thread and pack(batch, slot, staged) on a worker
    thread, two batches ahead of the compute; upload(batch, slot, packed) one batch ahead; compute(batch, slot, uploaded)
    enqueues batch k and returns a handle; finish(batch, handle) -> one result per image, called one batch behind, is the
    only stage that may wait for the device.  An exception of `batches` is raised after every batch before it has been
    yielded.  However the generator ends (exhausted, closed or raising), the worker thread is joined and drain() is
    called."""
    import concurrent.futures
    pool = concurrent.futures.ThreadPoolExecutor(max_workers=1, thread_name_prefix="ctpn-stream-pack")
    packing, uploaded = collections.deque(), collections.deque()
    state = {"k": 0, "error": None, "more": True}

    def pull():
        if not state["more"]:
            return
        try:
            batch = next(batches)
        except StopIteration:
            state["more"] = False
            return
        except Exception as e:
            state["more"], state["error"] = False, e
            return
        slot = state["k"] & 1
        state["k"] += 1
        packing.append((batch, slot, pool.submit(pack, batch, slot, stage(batch, slot))))

    def upload_next():
        if packing:
            batch, slot, fut = packing.popleft()
            uploaded.append((batch, slot, upload(batch, slot, fut.result())))

    ready, next_out, pending = {}, 0, None
    try:
        pull()
        upload_next()
        pull()
        while uploaded or pending is not None:
            this = None
            if uploaded:
                batch, slot, up = uploaded.popleft()
                this = (batch, compute(batch, slot, up))
                upload_next()
                pull()
            if pending is not None:
                for i, r in zip(pending[0].idxs, finish(*pending)):
                    ready[i] = r
                while next_out in ready:
                    yield ready.pop(next_out)
                    next_out += 1
            pending = this
        if state["error"] is not None:
            raise state["error"]
    finally:
        pool.shutdown(wait=True, cancel_futures=True)
        batches.close()
        drain()


# the 38 variables of the VGGnet_test graph (SURVEY.md App. A.2); a TF checkpoint also holds optimizer slots etc.
REQUIRED_VARIABLES = tuple(
    ["%s/%s" % (l, k) for l in ("conv1_1", "conv1_2", "conv2_1", "conv2_2", "conv3_1", "conv3_2", "conv3_3", "conv4_1",
                                "conv4_2", "conv4_3", "conv5_1", "conv5_2", "conv5_3", "rpn_conv/3x3")
     for k in ("weights", "biases")] +
    ["lstm_o/bidirectional_rnn/%s/lstm_cell/%s" % (d, k) for d in ("fw", "bw") for k in ("kernel", "bias")] +
    ["%s/%s" % (l, k) for l in ("lstm_o", "rpn_cls_score", "rpn_bbox_pred") for k in ("weights", "biases")])


def load_weight_file(path):
    """Weights from what the reference restores from, keyed by TF variable name:
      * a TF checkpoint V2 -- prefix, `.index` / `.data-*` file, or the directory holding the `checkpoint` state file
        (ctpn/demo.py:88-90: get_checkpoint_state + saver.restore),
      * a frozen GraphDef `.pb` (ctpn/generate_pb.py:36-40, ctpn/demo_pb.py),
      * the VGG `.npy` dict (network.py:40-53: np.load(..., encoding='latin1').item() -> {layer: {'weights', 'biases'}}),
      * this repo's `.npz` with those variable names.
    Checkpoints and graphs are reduced to the 38 network variables (a missing one raises KeyError)."""
    from . import tf_import
    if path.endswith(".npz"):
        with np.load(path) as z:
            return {k: z[k] for k in z.files}
    if path.endswith(".pb"):
        return {k: np.asarray(v, np.float32) for k, v in tf_import.read_frozen_graph(path, names=REQUIRED_VARIABLES).items()}
    if path.endswith(".npy"):
        d = np.load(path, allow_pickle=True, encoding="latin1").item()
        out = {}
        for layer, sub in d.items():
            for k, v in sub.items():
                out["%s/%s" % (layer, k)] = np.asarray(v, np.float32)
        return out
    prefix = tf_import.checkpoint_prefix(path)
    if not os.path.isfile(prefix + ".index"):
        raise FileNotFoundError("%s: not an .npz / .npy / .pb file and no TF checkpoint index at %s.index" % (path, prefix))
    return {k: np.asarray(v, np.float32) for k, v in tf_import.read_checkpoint(prefix, names=REQUIRED_VARIABLES).items()}
