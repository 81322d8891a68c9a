"""Engine: host-side driver of the H100 CTPN hot path.

PyTorch is used only as plumbing (device memory, streams, pinned buffers); all
compute is in libctpn_b200.so (see include/ctpn_b200.h).  One Engine == one GPU.

    eng = Engine(weights, planes=2)              # weights: {tf_variable_name: ndarray}
    scores, boxes = eng.detect(im)               # == lib.fast_rcnn.test.test_ctpn
    results = eng.detect_batch(uint8_batch)      # [B,H,W,3] -> list of (scores, boxes)
    results = eng.detect_ragged([im0, im1, ...])  # images of different sizes, batched on shared canvases
    results = eng.detect_images([photo0, ...])   # raw photos: resize_im + _get_image_blob on the device, then as above
    lines = eng.detect_lines_images([photo0, ...])  # ... and the text-line connector on the device: ctpn() per image

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
        kernel launches of a step cost more than the kernels themselves at batch 1); 0 disables graphs."""
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

    def _sizes_device(self, sizes, B, H, W, least=16, what="sizes"):
        """Per-image (h, w) of a ragged batch on its [B, H, W] canvas -> device int32 [B,2], checked on the host."""
        s = sizes.cpu().numpy() if torch.is_tensor(sizes) else np.asarray(sizes)
        s = np.asarray(s, np.int64).reshape(-1, 2) if s.size else s.reshape(0, 2)
        if s.shape != (B, 2):
            raise ValueError("%s: expected %d (h, w) pairs, got shape %s" % (what, B, tuple(np.shape(sizes))))
        if (s[:, 0] > H).any() or (s[:, 1] > W).any() or (s < least).any():
            raise ValueError("%s: every (h, w) must lie within the %dx%d canvas and be at least %d" % (what, H, W, least))
        return torch.from_numpy(s.astype(np.int32)).to(self.device, non_blocking=False)

    # ---- stages ----------------------------------------------------------------------------
    def forward_heads(self, images, ws_key="net", sizes=None):
        """images: CUDA tensor [B,H,W,3], uint8 BGR (mean subtraction fused) or float32 blob
        (already mean-subtracted, test.py:9).  Returns (rpn_cls_score [B,h,w,20] logits,
        rpn_bbox_pred [B,h,w,40]) float32 CUDA tensors.
        sizes: [B,2] (h, w) per image for a ragged batch (image b in rows < h and columns < w of its canvas slice, the rest
        ignored); each image's heads within (h >> 4, w >> 4) then equal a forward of that image alone.  None: uniform."""
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
            sz = self._sizes_device(sizes, B, H, W)
            N.check(N.lib.ctpn_net_forward_ragged(self._net, N.ptr(images), int(is_f32), N.ptr(sz), B, H, W, N.ptr(cls),
                                                  N.ptr(bbox), N.ptr(ws), ws.numel(), N.stream_ptr()), "ctpn_net_forward_ragged")
        return cls, bbox

    def recalibrate(self):
        """F16F8 mode: derive the activation scales again from the next batch (they are frozen after the first one).
        The scales put each layer's calibration maximum two binades below e4m3 saturation; activations beyond that saturate
        in the e4m3 copies, and those elements fall back to fp16 accuracy as long as they stay below 65504 / s in the fp16
        plane.  s is 1 unless the calibration maximum exceeds 2^14; a layer with s < 1 has only 2-3 binades of fp16 headroom,
        past which the element saturates in fp16 too and its error is unbounded.  So calibrate on representative images --
        not on a flat warm-up image -- and call this again when the input distribution changes."""
        N.check(N.lib.ctpn_net_set_option(self._net, b"recalibrate", 1), "set_option")
        self._graphs.clear()          # captured graphs hold the old scales as kernel arguments

    def tap(self, name):
        """Debug: float32 copy of a named activation of the last forward (keep_activations=True)."""
        cnt = C.c_size_t()
        N.check(N.lib.ctpn_net_debug_tap(self._net, name.encode(), None, 0, C.byref(cnt), None), "debug_tap")
        out = torch.empty(cnt.value, dtype=torch.float32, device=self.device)
        N.check(N.lib.ctpn_net_debug_tap(self._net, name.encode(), N.ptr(out), out.numel(), C.byref(cnt), N.stream_ptr()), "debug_tap")
        return out

    def proposals(self, cls, bbox, im_info, cls_is_logit=True, cfg=None, ws_key="prop", out=None, feat_sizes=None):
        """Batched proposal layer (proposal_layer_tf.py:14-157) on CUDA tensors.
        Returns rois [B,post,5] (score,x1,y1,x2,y2), index [B,post] int32, count [B] int32.
        out=(rois, count): write into these (contiguous) tensors instead of allocating.
        feat_sizes: [B,2] (fh, fw) per image of a ragged batch: only those cells of each image's heads are read, and index is
        image-local ((h * fw + w) * 10 + a).  None: every cell."""
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
            fs = self._sizes_device(feat_sizes, B, H, W, least=1, what="feat_sizes")
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

    def detect_packed(self, images, im_info, ws_tag="", sizes=None):
        """images: CUDA [B,H,W,3] uint8/float32; im_info: [B,3] tensor (blob_h, blob_w, scale).
        Returns ONE float32 device buffer [B*post*5 + B]: the rois of all images followed by the int32 counts
        (bit pattern), so that the D2H / the multi-GPU gather of a batch's results is a single transfer.
        sizes: [B,2] (h, w) per image of a ragged batch (see forward_heads), or None."""
        B = int(images.shape[0])
        if sizes is not None:
            sizes = np.asarray(sizes.cpu() if torch.is_tensor(sizes) else sizes, np.int64).reshape(-1, 2)
            feat = sizes >> 4
        rows = self.result_rows()
        packed = torch.empty(B * rows * 5 + B, dtype=torch.float32, device=self.device)
        rois, count = self.unpack(packed, B, rows)
        n = min(self.streams, B)
        if n <= 1:
            cls, bbox = self.forward_heads(images, ws_key="net" + ws_tag, sizes=sizes)
            self.proposals(cls, bbox, im_info, cls_is_logit=True, ws_key="prop" + ws_tag, out=(rois, count),
                           feat_sizes=None if sizes is None else feat)
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
                cls, bbox = self.forward_heads(images[lo:hi], ws_key="net%d" % i, sizes=None if sizes is None else sizes[lo:hi])
                self.proposals(cls, bbox, im_info[lo:hi], cls_is_logit=True, ws_key="prop%d" % i, out=(rois[lo:hi], count[lo:hi]),
                               feat_sizes=None if sizes is None else feat[lo:hi])
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

    def detect_lines_batches(self, batches, mode="H", im_info=None, workers=8, gather=False, cfg=None):
        """The whole ctpn() call chain (demo.py:55-68 minus file I/O) for a stream of host batches: rois_batches() on the
        GPU, then TextDetector.detect of every image in the library's host connector (ctpn_text_lines_host, which
        releases the GIL) on a pool of `workers` threads, one batch behind the GPU.  With gather=True (multi-GPU) the rois of
        all ranks are gathered as in rois_batches and every rank runs the connector on its own shard.  Yields, per batch, a list of
        float64 [m,9] text-line arrays (x1,y1,x2,y2,x3,y3,x4,y4,score) in the frame of the blob divided by im_scale."""
        from concurrent.futures import ThreadPoolExecutor
        from .textlines import text_lines

        def lines_of(rois, size, scale):
            return text_lines(rois[:, 1:5] / np.float32(scale), rois[:, 0], size, mode, cfg)

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
            H, W = shapes[k]
            scale = 1.0 if im_info is None else float(np.asarray(im_info, np.float32).reshape(-1, 3)[0, 2])
            futs = [pool.submit(lines_of, r, (int(round(H / scale)), int(round(W / scale))), scale) for r in rois_list]
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

    def rois_images(self, images, resize=True, max_batch=32, return_resized=False, scale=600, max_scale=1200):
        """The front half of ctpn() (demo.py:59-61) plus test_ctpn for a list of raw HxWx3 uint8 BGR images of any sizes,
        front-end on the device: resize_im (short side -> scale, long side <= max_scale; resize=False: the images are
        already at that scale) and _get_image_blob (uint8 when im_scale == 1, else the mean-subtracted float32 rescale),
        then ragged batches of at most max_batch (frontend_plan + ragged_plan).  Each batch's sources travel in one pinned
        H2D copy; ctpn_resize_linear_u8_ragged writes the uint8 canvas (or, for float32 batches, a uint8 canvas that
        ctpn_image_blob_f32_ragged turns into the float32 blob canvas), and detect_packed runs the batch with per-image
        extents.  Returns, in input order, (rois float32 [n,5] in blob coordinates, im_scale, f) per image -- and the
        resize_im output as a host uint8 array as a 4th item with return_resized (what draw_boxes draws on).  Every image
        is bit-identical to the host front-end with OpenCV's own code (IPP-dispatching cv2 builds differ on float
        rescales) followed by detect on that image alone.  Raises ValueError on a bad image (see frontend_plan)."""
        out = [None] * len(images)
        rows = self.result_rows()
        for idxs, items, out_h, resized in self._images_batches(images, resize, max_batch, return_resized, scale, max_scale,
                                                                "rois_images"):
            for k, (i, r) in enumerate(zip(idxs, self._split_results(out_h, len(idxs), rows))):
                out[i] = (r, items[k].im_scale, items[k].f) + ((resized[k],) if return_resized else ())
        return out

    def _images_batches(self, images, resize, max_batch, return_resized, scale, max_scale, what, after=None):
        """The batches of rois_images / detect_lines_images.  Per ragged batch: front-end, network and proposal layer on the
        device (detect_packed's buffer), then after(packed, items) -- device work enqueued on the rois, returning the buffer
        to bring back (None: the packed rois themselves) -- and one D2H of that buffer.  Yields (input indices, their
        FrontendSteps, the pinned host copy, the resize_im outputs or None); the pinned copy is reused by the next batch."""
        if not 1 <= int(max_batch) <= 64:
            raise ValueError("%s: max_batch must be 1..64 (the ragged front-end kernels take up to 64 images)" % what)
        images = [im.numpy() if torch.is_tensor(im) else np.asarray(im) for im in images]
        plan = frontend_plan(images, resize=resize, scale=scale, max_scale=max_scale, cfg=self.cfg)
        lut = self._mean_lut()
        stream = N.stream_ptr()
        for idxs, (H, W) in ragged_plan([p.blob for p in plan], [p.dtype for p in plan], max_batch):
            B = len(idxs)
            items = [plan[i] for i in idxs]
            nbytes = [images[i].size for i in idxs]
            offsets = np.cumsum([0] + nbytes[:-1]).astype(np.int64)
            total = int(sum(nbytes))
            pinned = self._pin("frontend_src", (1 << max(20, (total - 1).bit_length()),), torch.uint8)   # grow-only sizes
            pn = pinned.numpy()
            for k, i in enumerate(idxs):
                h, w = images[i].shape[:2]
                pn[offsets[k]:offsets[k] + nbytes[k]].reshape(h, w, 3)[...] = images[i]
            src = self._workspace("frontend_src", total)
            src[:total].copy_(pinned[:total], non_blocking=True)           # the batch's one H2D
            hwp = np.array([images[i].shape[:2] + (images[i].shape[1],) for i in idxs], np.int32)
            fxy = np.array([[p.f, p.f] for p in items], np.float64)
            is_u8 = items[0].dtype == "|u1"
            if is_u8:          # im_scale == 1: resize_im writes the network's uint8 canvas directly
                u8 = canvas = torch.empty((B, H, W, 3), dtype=torch.uint8, device=self.device)
                Hr, Wr = H, W
            else:
                Hr, Wr = max(p.resized[0] for p in items), max(p.resized[1] for p in items)
                u8 = self._workspace("frontend_u8", B * Hr * Wr * 3)[:B * Hr * Wr * 3].view(B, Hr, Wr, 3)
                canvas = torch.empty((B, H, W, 3), dtype=torch.float32, device=self.device)
            resized_hw = np.array([p.resized for p in items], np.int32)
            N.check(N.lib.ctpn_resize_linear_u8_ragged(N.ptr(src), total, N.ptr(offsets), N.ptr(hwp), N.ptr(fxy), N.ptr(resized_hw),
                                                       B, 3, N.ptr(u8), Hr, Wr, stream), "ctpn_resize_linear_u8_ragged")
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
            yield idxs, items, out_h, resized

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
                            cfg=None):
        """ctpn() (demo.py:55-68 minus file I/O) for a list of raw HxWx3 uint8 BGR images of any sizes, all on the device:
        the batches of rois_images (same inputs and batching), then the text-line connector (text_lines) on each batch's
        rois, and one D2H per batch of the packed lines, counts and statuses.  Returns, in input order, (lines float64
        [m,9] (x1,y1,x2,y2,x3,y3,x4,y4,score) in the resize_im frame, f) per image, plus the resize_im output with
        return_resized.  lines is bit-identical to TextDetector(native=True).detect(boxes, scores[:, None], resized.shape[:2])
        on detect_images' output for that image (mode "H" / "O" as cfg.TEST.DETECT_MODE; cfg: the 9 connector constants,
        None = text_connect_cfg's).  Raises CtpnError where that connector raises (a proposal outside the image width)."""
        if mode not in ("H", "O"):
            raise ValueError("mode must be 'H' or 'O' (got %r)" % (mode,))
        rows = self.result_rows()

        def connect(packed, items):
            B = len(items)
            rois, count = self.unpack(packed, B, rows)
            res = torch.empty(B * rows * 9 + B, dtype=torch.float64, device=self.device)
            self.text_lines(rois, count, [p.resized for p in items], [p.im_scale for p in items], mode, cfg,
                            out=self.unpack_lines(res, B, rows))
            return res

        out = [None] * len(images)
        for idxs, items, out_h, resized in self._images_batches(images, resize, max_batch, return_resized, scale, max_scale,
                                                                "detect_lines_images", after=connect):
            per_image = self.split_lines(*self.unpack_lines(out_h.numpy(), len(idxs), rows), im_hw=[p.resized for p in items])
            for k, (i, lines) in enumerate(zip(idxs, per_image)):
                out[i] = (lines, items[k].f) + ((resized[k],) if return_resized else ())
        return out

    def detect_images(self, images, resize=True, max_batch=32, return_resized=False, scale=600, max_scale=1200):
        """rois_images as test_ctpn returns it: per image (scores float32 [n], boxes float64 [n,4] = rois / im_scale, f), plus
        the resize_im output with return_resized.  Boxes are in the resize_im frame, as TextDetector expects them
        (draw_boxes divides by f)."""
        res = self.rois_images(images, resize=resize, max_batch=max_batch, return_resized=return_resized, scale=scale,
                               max_scale=max_scale)
        return [(r[0][:, 0], r[0][:, 1:5] / np.float64(r[1])) + tuple(r[2:]) for r in res]

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


FrontendStep = collections.namedtuple("FrontendStep", "f resized im_scale blob dtype")


def _cv_round_size(h, w, s):
    return int(np.rint(float(h) * s)), int(np.rint(float(w) * s))        # cvRound: round half to even, in float64


def frontend_plan(shapes, resize=True, scale=600, max_scale=1200, cfg=None):
    """What the demo's host front-end does to each image, computed on the host: shapes is a list of HxWx3 uint8 images
    (anything with .shape and .dtype) or of (H, W[, 3]) tuples.  Per image a FrontendStep of
      f         the resize_im factor (ctpn/demo.py: short side -> scale unless the long side would exceed max_scale;
                1.0 with resize=False, for images already at that scale),
      resized   its (h, w) as cv2.resize computes it (cvRound),
      im_scale  _get_image_blob's scale (lib/fast_rcnn/test.py _im_scale: SCALES[0] / short side, or MAX_SIZE / long side
                when np.round(im_scale * long side) > MAX_SIZE; cfg: SCALES and MAX_SIZE, default DEFAULT_CFG),
      blob      the (h, w) of the blob the network sees,
      dtype     '|u1' when im_scale == 1 (the uint8 image is the blob), else '<f4' (the float32 rescale).
    Raises ValueError when an image is not HxWx3 uint8, a resize would be empty or a blob side would be under 16."""
    c = dict(DEFAULT_CFG)
    if cfg:
        c.update(cfg)
    target, max_size = float(c["SCALES"][0]), float(c["MAX_SIZE"])
    out = []
    for i, s in enumerate(shapes):
        if hasattr(s, "shape") and hasattr(s, "dtype"):
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
        out.append(FrontendStep(f, (rh, rw), im_scale, (bh, bw), "|u1" if im_scale == 1.0 else "<f4"))
    return out


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
