/*
 * ctpn_b200 -- C ABI of the H100-native (sm_90a) CTPN detection hot path.
 *
 * One shared library (libctpn_b200.so, nvcc -gencode arch=compute_90a,code=sm_90a),
 * plain pointers and sizes only, no torch / C++ types.  Every entry point returns an
 * int status (0 = success); ctpn_last_error() gives the message for the calling thread.
 * Unless a name ends in _host, pointers are DEVICE pointers on the current device and
 * `stream` is a cudaStream_t passed as void*.  No entry point allocates device memory
 * except ctpn_nms_host (grow-only per-device scratch) and ctpn_net_* weight storage.
 *
 * Reference interfaces replaced (paths relative to eragonruan/text-detection-ctpn @ c04a571e):
 *   ctpn_nms_host        lib/utils/gpu_nms.hpp:1-2  `void _nms(int*,int*,const float*,int,int,float,int)`
 *                        (called by lib/utils/gpu_nms.pyx:31)
 *   ctpn_nms_sorted      lib/utils/nms_kernel.cu:34-78 (nms_kernel) + :124-139 (host greedy scan)
 *   ctpn_proposals       lib/rpn_msr/proposal_layer_tf.py:14-157 (tf.py_func body, lib/networks/network.py:214)
 *   ctpn_conv1_1_tc[_f16f8] / ctpn_conv3x3[_f16f8] (taps=9, optional fused 2x2 max-pool)
 *                        lib/networks/network.py:160-183 (conv), :189-196 (max_pool)
 *   ctpn_bilstm_recurrent, ctpn_conv3x3 (taps=1: x-projection, FC and head matmuls)
 *                        lib/networks/network.py:88-113 (Bilstm), :144-158 (lstm_fc)
 *   ctpn_net_forward     lib/networks/VGGnet_test.py:16-52 up to the two head tensors
 *                        (the demo_pb.py:73-75 boundary), fed by lib/fast_rcnn/test.py:7-31
 *   ctpn_resize_linear_u8   cv2.resize in resize_im, ctpn/demo.py:21-25 (and draw_boxes :50)
 *   ctpn_image_blob_f32     _get_image_blob, lib/fast_rcnn/test.py:7-31 (float32 cv2.resize of the mean-subtracted image)
 *   ctpn_resize_linear_u8_ragged / ctpn_image_blob_f32_ragged   the same two, for a batch of images of different sizes
 *   ctpn_resize_linear_u8_ragged_rows     the ragged resize on sources that hold only the rows it reads
 *   ctpn_resize_linear_u8_strided         the ragged resize on images read in place at any byte strides
 *   ctpn_resize_linear_u8_yuv420          the same on YUV 4:2:0 frames, with cv2.cvtColor's conversion to BGR
 *   ctpn_text_filter_nms_host / ctpn_text_groups_host / ctpn_text_lines_host / ctpn_text_lines (batched, device)
 *                        TextDetector.detect, lib/text_connector/detectors.py:19-49; graph builder
 *                        text_proposal_graph_builder.py:6-78; chains other.py:16-29; line fitting
 *                        text_proposal_connector.py:21-64 and text_proposal_connector_oriented.py:24-105
 *   ctpn_line_crop_widths_host / ctpn_line_crops_u8   the recognizer's line crops (cv2.warpAffine) a user would otherwise
 *                        cut from draw_boxes' image on the host
 *   ctpn_line_crops_strided_u8 / ctpn_line_crops_yuv420_u8   the same crops out of the source images at full resolution
 *   ctpn_bbox_overlaps_host / ctpn_bbox_intersections_host   lib/utils/bbox.pyx:15-55, :57-95 (Cython, CPU)
 *   ctpn_anchor_targets_host   lib/rpn_msr/anchor_target_layer_tf.py:78-175, :201 (tf.py_func body, network.py:225-243;
 *                        training only -- host code, as the reference's is)
 *   ctpn_crc32c_host     the per-tensor checksum of the TF checkpoints the reference restores (ctpn/demo.py:88-90)
 * Test-only entry points (float32 SIMT reference kernels, hardware probes) and every ablation / tuning switch are NOT in
 * this library: they live in tests/_native/libctpn_b200_dbg.so (csrc/testing/ctpn_b200_testing.h).
 */
#ifndef CTPN_B200_H_
#define CTPN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CTPN_OK 0
#define CTPN_ERR_INVALID 1   /* bad argument */
#define CTPN_ERR_CUDA 2      /* CUDA runtime / driver error */
#define CTPN_ERR_WORKSPACE 3 /* workspace too small */
#define CTPN_ERR_NO_DEVICE 4 /* no usable sm_90 device */

/* ---- library ------------------------------------------------------------------------- */
int ctpn_version(void);                 /* 10000*major + 100*minor + patch */
const char *ctpn_last_error(void);      /* thread-local, never NULL */
int ctpn_device_ok(int device_id);      /* CTPN_OK iff device exists and is compute capability 10.x */

/* Per-launch timing with CUDA events on the launching stream (used by bench.py for the roofline
 * numbers).  ctpn_prof_enable(1) clears and starts recording, (0) stops.  ctpn_prof_report
 * synchronises the recorded events and writes a JSON array
 *   [{"kernel": label, "launches": n, "ms": total, "work": algorithmic FLOPs}, ...]
 * into buf (if capacity allows); *needed receives the required size including the NUL. */
int ctpn_prof_enable(int on);
int ctpn_prof_report(char *buf, size_t capacity, size_t *needed);

/* ---- NMS ------------------------------------------------------------------------------
 * ctpn_nms_host: drop-in for `_nms`.  All pointers are HOST memory.  boxes_host is row
 * major [boxes_num, boxes_dim] (boxes_dim >= 4, columns x1,y1,x2,y2,...), already sorted by
 * score descending.  keep_out must hold boxes_num ints; *num_out receives the count.
 * Suppression rule: IoU(+1 pixel convention, float32, no FMA contraction) > thresh.
 * Unlike `_nms` it returns a status instead of printing CUDA errors and carrying on. */
int ctpn_nms_host(int *keep_out, int *num_out, const float *boxes_host, int boxes_num,
                  int boxes_dim, float nms_overlap_thresh, int device_id);

/* Batched device NMS over pre-sorted boxes.  boxes: [batch][max_n][4] float; counts[batch]
 * gives the valid prefix of each image.  keep_out: [batch][max_keep] positions (ascending),
 * num_out[batch].  max_keep > 0 stops the greedy scan early (proposal_layer_tf.py:145-146). */
size_t ctpn_nms_workspace_bytes(int batch, int max_n);
int ctpn_nms_sorted(const float *boxes, const int *counts, int batch, int max_n, float thresh,
                    int max_keep, int *keep_out, int *num_out, void *workspace,
                    size_t workspace_bytes, void *stream);

/* ---- proposal layer (batched; per-image semantics == the reference's batch-1 layer) ---
 * cls:  [batch][H][W][20]  softmax probabilities (cls_is_logit=0, the demo_pb.py boundary)
 *                          or raw rpn_cls_score logits (cls_is_logit=1; pair softmax fused)
 * bbox: [batch][H][W][40]  (dx,dy,dw,dh) per anchor
 * im_info: [batch][3]      (blob_h, blob_w, im_scale)
 * rois_out:  [batch][post_nms_topN][5] = (score,x1,y1,x2,y2), rows past the count are 0
 * index_out: [batch][post_nms_topN]    flat (h,w,a) anchor index of each row (may be NULL)
 * count_out: [batch]
 * anchors_py2 != 0 selects the Python-2 anchor table (SURVEY.md App. A.3). */
size_t ctpn_proposals_workspace_bytes(int batch, int H, int W, int pre_nms_topN);
int ctpn_proposals(const float *cls, int cls_is_logit, const float *bbox, const float *im_info,
                   int batch, int H, int W, int feat_stride, int pre_nms_topN, int post_nms_topN,
                   float nms_thresh, float min_size, int anchors_py2, float *rois_out,
                   int *index_out, int *count_out, void *workspace, size_t workspace_bytes,
                   void *stream);
/* Ragged batch (see ctpn_net_forward_ragged): feat_hw (device int32 [batch][2]) is each image's feature-map size (fh, fw)
 * within the H x W canvas of the head tensors.  Anchors of cells outside it are never valid and their head values are
 * never read; index_out is image-local, (h * fw + w) * 10 + a.  Per image the result is that of ctpn_proposals on the image's
 * own fh x fw heads.  Same workspace as ctpn_proposals for (batch, H, W). */
int ctpn_proposals_ragged(const float *cls, int cls_is_logit, const float *bbox, const float *im_info, const int *feat_hw,
                          int batch, int H, int W, int feat_stride, int pre_nms_topN, int post_nms_topN, float nms_thresh,
                          float min_size, int anchors_py2, float *rois_out, int *index_out, int *count_out,
                          void *workspace, size_t workspace_bytes, void *stream);

/* ---- network stages --------------------------------------------------------------------
 * Activation format ("planes"): P in {1,2,3} bf16 tensors [P][B][H][W][C] whose element-wise
 * sum is the float32 value (a = a1 + a2 (+ a3), a1 = bf16(a), a2 = bf16(a - a1), ...).
 * P=1 is plain bf16, P=3 carries all 24 mantissa bits.  Products of planes are accumulated
 * in float32 on the tensor cores (wgmma, register accumulators).
 * Weight format: bf16 [P][Cout][taps][Cin] (K-major), made by ctpn_pack_weights from the
 * TF layout [taps][Cin][Cout] (HWIO for 3x3, [K][N] for matmuls). */
int ctpn_pack_weights(const float *w_tf, int taps, int cin, int cout, int cout_pad, int planes,
                      void *w_planes_out, void *stream);

/* conv1_1: uint8 BGR image [B][H][W][3] (or float32 blob when src_is_f32) -> 64-channel planes; fuses the mean
 * subtraction of lib/fast_rcnn/test.py:9 (lut[256][3] = float32(double(v) - PIXEL_MEANS[c])), bias and ReLU.  On the
 * tensor cores: the im2col tile (K = 27 padded to 32) is built in shared memory as bf16 planes and multiplied by the
 * resident weight tile with wgmma; HBM-write bound. */
int ctpn_conv1_1_tc(const void *src, int src_is_f32, const float *lut, const float *w_hwio,
                    const float *bias, void *out_planes, int B, int H, int W, int planes, void *stream);

/* 3x3 SAME conv (taps=9) or 1x1 / matmul (taps=1) on planes with wgmma tensor cores.
 * flags: bit0 ReLU, bit1 fused 2x2/2 VALID max-pool (taps=9 only), bit2 float32 output
 * [B][H][W][Cout] instead of planes.  Cin % 64 == 0, Cout % 64 == 0. */
#define CTPN_F_RELU 1
#define CTPN_F_POOL 2
#define CTPN_F_OUT_F32 4
#define CTPN_F_OUT_BF16X2 8 /* ctpn_conv3x3_f16f8 only: write two bf16 planes instead of F16F8 planes */
/* Row-stacked batches: a tensor [B][H + 1][W][C] with one ZERO row after every image is one tall image for the tiling (a 37-row
 * map wastes 23 % of its 16-row tiles, a 32 x 38-row stack none) while the zero rows keep the images' halos apart.
 * STACK_IN: the input is stacked (taps = 9, no pooling; H is still the image height).  STACK_OUT: write the output in the
 * stacked layout [B][Ho + 1][Wo] -- a STACK_IN layer also writes the zero rows, a plain-input layer leaves them to the caller. */
#define CTPN_F_STACK_IN 16
#define CTPN_F_STACK_OUT 32
/* PROMOTE (ctpn_conv3x3 with planes = 3 only; CTPN_ERR_INVALID otherwise and on ctpn_conv3x3_f16f8): the tensor core truncates
 * when it adds a K=16 partial sum into a float32 accumulator, and over the 9 * Cin / 16 adds of a 512-channel layer those
 * truncations add up to ~10x the error of float32 with round-to-nearest (DESIGN.md section 5).  With this flag the plane-0 x
 * plane-0 accumulator restarts every 64 channels of one tap and its partial sums are added with round-to-nearest float32
 * adds; the cross-plane terms (2^-8 smaller) accumulate as before. */
#define CTPN_F_PROMOTE 64
int ctpn_conv3x3(const void *in_planes, const void *w_planes, const float *bias, void *out, int B,
                 int H, int W, int cin, int cout, int taps, int planes, int flags, void *stream);
/* The same layers in the "F16F8" arithmetic: 2 tensor-core units per MAC instead of the 3 of two bf16 planes; head logits
 * within 1e-3 of float32 (DESIGN.md section 5).  A value a is carried as h = fp16(a * s) plus e4m3 copies of a and of the exact
 * residual a * s - h; products are h_a * h_w on fp16 MMAs plus the two cross terms on e4m3 MMAs.
 * Activation planes: [0] fp16 [B][H][W][C]; [1] per pixel and 64-channel block 128 bytes e4m3(a * t)[64] | e4m3(r * 2^11 t / s)[64].
 * Weight planes (ctpn_pack_weights_f16f8): [0] fp16(w * s_w) [Cout][taps][Cin]; [1] per (cout, tap, 64-channel block)
 * e4m3(r_w * 2^11 t_w / s_w)[64] | e4m3(w * t_w)[64].  All scales are powers of two chosen by the caller (per tensor).
 * ctpn_conv3x3_f16f8: value = main * inv_main + cross * inv_cross with inv_main = 1 / (s_in * s_w) and
 * inv_cross = 1 / (2^11 * t_in * t_w); outputs are quantised with out_s / out_t (F16F8 planes), or written as float32
 * (CTPN_F_OUT_F32) or as two bf16 planes (CTPN_F_OUT_BF16X2).  Same shape rules and flags as ctpn_conv3x3. */
int ctpn_pack_weights_f16f8(const float *w_tf, int taps, int cin, int cout, int cout_pad, float s_w, float t_w,
                            void *w_planes_out, void *stream);
int ctpn_conv3x3_f16f8(const void *in_planes, const void *w_planes, const float *bias, void *out, int B, int H, int W,
                       int cin, int cout, int taps, int flags, float inv_main, float inv_cross, float out_s, float out_t,
                       void *stream);

/* conv1_1 writing F16F8 planes (the layer itself multiplies two bf16 planes; K = 27). */
int ctpn_conv1_1_tc_f16f8(const void *src, int src_is_f32, const float *lut, const float *w_hwio, const float *bias,
                          void *out_planes, int B, int H, int W, float out_s, float out_t, void *stream);

/* BiLSTM recurrence (network.py:97-101).  xproj: float32 [R][W][1024] = x.Wx + b for
 * (fw gates i,j,f,o | bw gates i,j,f,o); wh_fw / wh_bw: float32 [128][512] recurrent kernels
 * (rows 512..639 of the TF kernel).  Output planes [P][R][W][256] = concat(h_fw, h_bw). */
int ctpn_bilstm_recurrent(const float *xproj, const float *wh_fw, const float *wh_bw,
                          void *out_planes, int R, int W, int planes, void *stream);

/* ---- whole network up to the head tensors -------------------------------------------- */
typedef struct ctpn_net ctpn_net_t;
/* planes: 1..3 bf16 planes, CTPN_ARITH_BF16X3P, or CTPN_ARITH_F16F8: conv1_1 + the thirteen 3x3 layers in the 2-unit F16F8 arithmetic (the
 * matmuls around the BiLSTM stay on two bf16 planes).  F16F8 activation scales are calibrated on the first batch that
 * ctpn_net_forward sees and then frozen (option "recalibrate" re-arms the calibration).
 * CTPN_ARITH_BF16X3P: three bf16 planes (as planes = 3) with CTPN_F_PROMOTE on the thirteen 3x3 layers and the three matmuls
 * (x-projection, FC, heads); conv1_1 (K = 32, one two-MMA chain) and the BiLSTM are the same as with planes = 3. */
#define CTPN_ARITH_F16F8 4
#define CTPN_ARITH_BF16X3P 5
int ctpn_net_create(ctpn_net_t **net, int planes);
int ctpn_net_destroy(ctpn_net_t *net);
/* options: "keep_activations" (1: every layer gets its own workspace region so that
 * ctpn_net_debug_tap can read all of them after a forward), "recalibrate" (F16F8: re-derive the activation scales from
 * the next batch). */
int ctpn_net_set_option(ctpn_net_t *net, const char *key, int value);
/* name = TF variable name (SURVEY.md App. A.2); data = host float32 in TF layout. */
int ctpn_net_set_weight(ctpn_net_t *net, const char *name, const float *data_host, size_t count);
size_t ctpn_net_workspace_bytes(const ctpn_net_t *net, int B, int H, int W);
/* images: uint8 [B][H][W][3] BGR (device).  Outputs (device, float32):
 * cls_score [B][H/16][W/16][20] logits, bbox_pred [B][H/16][W/16][40]. */
int ctpn_net_forward(ctpn_net_t *net, const void *images, int src_is_f32, int B, int H, int W,
                     float *cls_score_out, float *bbox_pred_out, void *workspace,
                     size_t workspace_bytes, void *stream);
/* Ragged batch: B images of different sizes on one canvas [B][H][W][3]; image b occupies rows < h_b and columns < w_b of its
 * slice (sizes: device int32 [B][2] = (h_b, w_b), 16 <= h_b <= H, 16 <= w_b <= W; a size beyond the canvas is clamped to it).
 * The canvas outside an image is never read.  Every layer stores exact zeros outside the image's extent at its level,
 * (h_b >> k, w_b >> k) after k pools, which the next 3x3 layer takes as its SAME padding; so each image's head tensors within
 * (h_b >> 4, w_b >> 4) equal ctpn_net_forward of that image alone, bit for bit, in every arithmetic.  The head values outside
 * that extent are unspecified.  Workspace: ctpn_net_workspace_bytes(net, B, H, W). */
int ctpn_net_forward_ragged(ctpn_net_t *net, const void *images, int src_is_f32, const int *sizes, int B, int H, int W,
                            float *cls_score_out, float *bbox_pred_out, void *workspace, size_t workspace_bytes,
                            void *stream);
/* feature-map size after the four VALID pools */
int ctpn_net_feature_hw(int H, int W, int *fh, int *fw);
/* Debug tap: copies the most recent forward's named activation ("conv1_1" ... "rpn_conv/3x3",
 * "lstm_out", "lstm_o") to out_f32 (device float32, NHWC).  Returns element count via *count. */
int ctpn_net_debug_tap(ctpn_net_t *net, const char *name, float *out_f32, size_t capacity,
                       size_t *count, void *stream);

/* ---- image front-end (replaces cv2.resize in resize_im, ctpn/demo.py:21-25) ----
 * cv2.resize(src, None, None, fx, fy, INTER_LINEAR) for uint8 [B][sh][sw][channels] device images, bit-exact with
 * OpenCV's fixed-point path (incl. its INTER_AREA routing of an exact 1/2 scale).  ctpn_resize_out_size gives the
 * destination size cv2 would produce (cvRound(src * f)); dst must have exactly that size. */
int ctpn_resize_out_size(int sh, int sw, double fx, double fy, int *dh, int *dw);
int ctpn_resize_linear_u8(const void *src, int B, int sh, int sw, int channels, double fx, double fy, void *dst, int dh,
                          int dw, void *stream);

/* The float32 rescale of _get_image_blob (lib/fast_rcnn/test.py:7-31) fused with the mean subtraction: uint8 BGR
 * [B][sh][sw][3] -> float32 blob [B][dh][dw][3] = cv2.resize(float32(im) - PIXEL_MEANS, fx, fy, INTER_LINEAR) as OpenCV's own
 * float code computes it (bit-exact; opencv-python builds that dispatch to Intel IPP differ from that by up to ~1.4e-2 on 8-bit-range data).
 * lut[256][3] = float32(double(v) - PIXEL_MEANS[c]) (device).  dst size from ctpn_resize_out_size. */
int ctpn_image_blob_f32(const void *src_u8, const float *lut, int B, int sh, int sw, double fx, double fy, float *dst, int dh,
                        int dw, void *stream);

/* Ragged forms of the two calls above: B images of different sizes and scales in one launch.  Image b is read from
 * src + src_offset[b] (elements) as [h][pitch][C] with (h, w, pitch) = src_hwp[3b..3b+2] (pitch >= w pixels per row),
 * resized by (fx, fy) = fxy[2b..2b+1] to dst_hw[2b..2b+1] (must equal ctpn_resize_out_size), and written to rows < dh,
 * columns < dw of slice b of the canvas dst [B][H][W][C]; the rest of the canvas is NOT written.  Every image is
 * bit-identical to the single-image call on that image alone (same per-pixel code, incl. the INTER_AREA routing of an
 * exact 1/2 scale).  ctpn_image_blob_f32_ragged: C = 3, float32 canvas, lut as for ctpn_image_blob_f32.
 * EXCEPTION to the pointer convention of this header: src_offset, src_hwp, fxy and dst_hw are small HOST arrays
 * (1 <= B <= 64); src, dst and lut are device pointers, src_elems the number of elements src holds.  Every descriptor is
 * validated before any CUDA call (CTPN_ERR_INVALID naming the image: dst_hw != cvRound size, output larger than the
 * canvas, offset + ((h - 1) * pitch + w) * C > src_elems, pitch < w, a scale <= 0, a NULL pointer) and then passed to
 * the kernel by value, so the kernel touches no memory whose extent the host did not check. */
int ctpn_resize_linear_u8_ragged(const void *src, size_t src_elems, const long long *src_offset, const int *src_hwp,
                                 const double *fxy, const int *dst_hw, int B, int channels, void *dst, int H, int W,
                                 void *stream);
int ctpn_image_blob_f32_ragged(const void *src_u8, size_t src_elems, const long long *src_offset, const int *src_hwp,
                               const double *fxy, const int *dst_hw, const float *lut, int B, float *dst, int H, int W,
                               void *stream);

/* ctpn_resize_linear_u8_ragged for row-compacted sources: INTER_LINEAR reads two source rows per output row, so a strong
 * downscale (f = 0.2: 2 of every 5 rows) leaves most rows unread, and a caller that uploads the images need not send
 * them.  Image b is [stored_rows[b]][pitch][C] at src + src_offset[b]: a subset of the rows of the (h, w) = src_hwp image,
 * in ascending order, holding at least every row the resize reads.  row_map (DEVICE int32, map_elems entries) holds, at
 * map_offset[b], one entry per ORIGINAL row y < h: the stored index of row y (any value for rows that are not stored;
 * the identity for an image stored densely, which an exact 1/2 scale must be: its INTER_AREA route reads every row).
 * Taps, weights, border clamping and the output size come from the original (h, w) exactly as in the dense call -- the
 * same per-pixel code -- and only the row address goes through the map, so with a correct map every image is bit-identical
 * to ctpn_resize_linear_u8_ragged on the full image.  stored_rows and map_offset are HOST arrays like the other
 * descriptors.  Validated before any CUDA call, in addition to the dense call's checks (CTPN_ERR_INVALID naming the
 * image): 1 <= stored_rows <= h, offset + ((stored_rows - 1) * pitch + w) * C <= src_elems, map_offset >= 0 and
 * map_offset + h <= map_elems.  The map's CONTENT is not trusted: the kernel clamps every entry to [0, stored_rows), so
 * a wrong map gives wrong pixels, never a read outside the extent that was checked. */
int ctpn_resize_linear_u8_ragged_rows(const void *src, size_t src_elems, const long long *src_offset, const int *src_hwp,
                                      const int *stored_rows, const int *row_map, size_t map_elems, const long long *map_offset,
                                      const double *fxy, const int *dst_hw, int B, int channels, void *dst, int H, int W,
                                      void *stream);

/* ctpn_resize_linear_u8_ragged for images read in place from memory the caller owns (e.g. device tensors of any strides):
 * image b is the (h, w) = src_hw[2b..2b+1] uint8 image whose sample (y, x, c) lies at byte
 *   src[b] + src_offset[b] + y * src_strides[3b] + x * src_strides[3b + 1] + c * src_strides[3b + 2]
 * of the allocation src[b] (a DEVICE address) of src_bytes[b] bytes.  Strides are signed and may be zero, so channel
 * order and planar layouts are strides too: an RGB image is read as BGR from channel 2 with a negative channel stride.
 * The 3-channel output is written exactly as ctpn_resize_linear_u8_ragged writes it (rows < dh, columns < dw of slice b of
 * dst [B][H][W][3]; the rest NOT written), bit-identical to it on a dense BGR copy of the image.  src, src_bytes,
 * src_offset, src_strides, src_hw, fxy and dst_hw are HOST arrays (1 <= B <= 64).  Validated before any CUDA call, with
 * the size, scale, dst_hw and canvas rules of ctpn_resize_linear_u8_ragged and in addition (CTPN_ERR_INVALID naming the
 * image): a NULL src[b]; the lowest and the highest byte the h x w x 3 box can touch must lie in [0, src_bytes[b]); the
 * column and channel strides must fit in 32 bits. */
int ctpn_resize_linear_u8_strided(const void *const *src, const size_t *src_bytes, const long long *src_offset,
                                  const long long *src_strides, const int *src_hw, const double *fxy, const int *dst_hw, int B,
                                  void *dst, int H, int W, void *stream);

/* ctpn_resize_linear_u8_strided for YUV 4:2:0 frames read in place (e.g. NV12 surfaces of a video decoder): image b is
 * the (h, w) = src_hw[2b..2b+1] frame whose planes p = 0, 1, 2 (Y, U, V) have their sample (y, x) at byte
 *   planes[3b + p] + plane_offset[3b + p] + y * plane_strides[6b + 2p] + x * plane_strides[6b + 2p + 1]
 * of the allocation planes[3b + p] (a DEVICE address) of plane_bytes[3b + p] bytes; Y is h x w, U and V are h/2 x w/2.
 * Strides are signed and may be zero, so NV12 / NV21 (interleaved chroma: column stride 2, U and V one byte apart), I420 /
 * YV12, pitched surfaces, planes in separate allocations and even-offset crops are all descriptors.  Each sample is
 * converted to BGR as cv2.cvtColor(COLOR_YUV2BGR_NV12 / _NV21 / _I420 / _YV12) converts it (BT.601 limited range, 20-bit
 * fixed point, nearest chroma), then resized as ctpn_resize_linear_u8_strided resizes; the output, written exactly as that
 * call writes it, is bit-identical to it on the cvtColor output.  planes, plane_bytes, plane_offset, plane_strides,
 * src_hw, fxy and dst_hw are HOST arrays (1 <= B <= 64).  Validated before any CUDA call, with the size, scale, dst_hw and
 * canvas rules of ctpn_resize_linear_u8_ragged and in addition (CTPN_ERR_INVALID naming the image and the plane): h and w
 * even; a NULL plane; the lowest and the highest byte each plane's box can touch must lie in [0, plane_bytes); column
 * strides must fit in 32 bits. */
int ctpn_resize_linear_u8_yuv420(const void *const *planes, const size_t *plane_bytes, const long long *plane_offset,
                                 const long long *plane_strides, const int *src_hw, const double *fxy, const int *dst_hw,
                                 int B, void *dst, int H, int W, void *stream);

/* CRC-32C (Castagnoli) of a host buffer, continuing from `crc` (0 to start): the per-tensor checksum of TF checkpoint V2
 * files, used by the weight importer (ctpn_b200/tf_import.py) to verify every tensor it loads. */
uint32_t ctpn_crc32c_host(const void *data, size_t n, uint32_t crc);

/* ---- text lines (replaces lib/text_connector/detectors.py:19-49 and the connector classes) ----
 * Two connectors with one arithmetic (csrc/textline.cuh: the same __host__ __device__ functions, no FMA contraction, IEEE
 * division and sqrt): ctpn_text_lines_host on the CPU for one image, ctpn_text_lines on the device for a batch.  Their
 * lines are equal as float64 bits.
 *
 * ctpn_text_lines: the connector for a batch of the proposal layer's outputs, where they lie on the device.
 *   rois [batch][rows][5] (score, x1, y1, x2, y2) in blob coordinates and counts [batch] (valid rows per image) are device
 *   arrays in ctpn_proposals' layout; the rows may come in any order.  im_hw [batch][2] (h, w: the frame of the lines, i.e.
 *   the resize_im output) and im_scale [batch] (the blob scale) are small HOST arrays (1 <= batch <= 64), validated
 *   before any CUDA call.  For every image b, num_lines[b] and the first num_lines[b] rows of lines_out[b] ([batch][rows][9]
 *   float64, device) equal ctpn_text_lines_host on boxes = float32(double(roi[1:5]) / im_scale[b]) (test_ctpn's
 *   rois / np.float64(im_scale) stored as float32), scores = roi[0], size im_hw[b], with the same oriented and cfg9.
 *   Rows of lines_out[b] past num_lines[b] are not written.  Every line starts at a distinct chain head, which is one of
 *   the counts[b] <= rows proposals, so rows lines per image always suffice.
 *   status [batch] (device): 0, 1 where ctpn_text_lines_host would fail because a surviving proposal's x1 lies outside
 *   [0, w) (the reference raises IndexError; the kernel never reads outside its column table), 2 where counts[b] is not
 *   in [0, rows]; num_lines[b] is 0 for a nonzero status and the other images are unaffected.
 *   0 <= rows <= 65536; every per-image array lives in the workspace (ctpn_text_lines_workspace_bytes(batch, rows, max w),
 *   O(rows^2 / 8) bytes per image for the NMS bitmask), CTPN_ERR_INVALID when it is smaller or an argument is bad.
 *   Stream-ordered, no allocation, no synchronisation; CTPN_ERR_NO_DEVICE without a GPU.
 *
 * ctpn_text_lines_host: TextDetector.detect in C++ on the CPU: score filter (> 0.7), score order, NMS 0.2, proposal graph
 * (text_proposal_graph_builder.py:6-78), chains (other.py:16-29), horizontal (oriented = 0,
 * text_proposal_connector.py:13-64) or oriented (1, text_proposal_connector_oriented.py:24-105) line fitting and
 * filter_boxes.  proposals [n][4] and scores [n] are test_ctpn()'s output (host memory); lines_out receives
 * *num_lines rows of 9 doubles (x1,y1,x2,y2,x3,y3,x4,y4,score).  cfg9 = NULL for text_connect_cfg.py's constants, else
 * (min_score, nms_thresh, max_gap, min_v_overlaps, min_size_sim, min_ratio, line_min_score, proposal_width,
 * min_num_proposals).  CTPN_ERR_INVALID (with *num_lines set) when more than max_lines lines were found. */
int ctpn_text_lines_host(const float *proposals, const float *scores, int n, int im_h, int im_w, int oriented,
                         const float *cfg9, double *lines_out, int max_lines, int *num_lines);
size_t ctpn_text_lines_workspace_bytes(int batch, int rows, int max_im_w);
int ctpn_text_lines(const float *rois, const int *counts, int batch, int rows, const int *im_hw, const double *im_scale,
                    int oriented, const float *cfg9, double *lines_out, int *num_lines, int *status, void *workspace,
                    size_t workspace_bytes, void *stream);

/* The stages of ctpn_text_lines_host for callers that fit the lines themselves (the Python TextDetector mirror fits with
 * numpy so that np.polyfit's own LAPACK solve produces the coordinates).
 * ctpn_text_filter_nms_host: detectors.py:21-28 -- score filter, score order (index ascending on ties), greedy NMS;
 * keep_out[n] receives *num_keep indices into the input, in visiting order.
 * ctpn_text_groups_host: graph + chain walk over m proposals in the given order (what get_text_lines receives);
 * chain g = members[offsets[g] .. offsets[g+1]), offsets[m+1].  Chains that run into the same successor share their
 * tails, so *num_members can exceed m: CTPN_ERR_WORKSPACE (with *num_members set) when members_capacity is too small. */
int ctpn_text_filter_nms_host(const float *proposals, const float *scores, int n, const float *cfg9, int *keep_out,
                              int *num_keep);
int ctpn_text_groups_host(const float *proposals, const float *scores, int m, int im_w, const float *cfg9, int *offsets,
                          int *members, int members_capacity, int *num_groups, int *num_members);

/* ---- text-line crops (the input of a line recognizer) ----
 * The crop of a line [x1,y1,x2,y2,x3,y3,x4,y4,score] (corners TL, TR, BL, BR, in the resize_im frame) at height hc
 * (2 <= hc <= 256) is cv2.warpAffine(resized, Minv, (Wc, hc), INTER_LINEAR | WARP_INVERSE_MAP, BORDER_REPLICATE) with
 *   len = sqrt((x2-x1)^2 + (y2-y1)^2), ht = sqrt((x3-x1)^2 + (y3-y1)^2), Wc = max(2, rint(hc * len / max(ht, 1)))
 *   Minv = [[(x2-x1)/(Wc-1), (x3-x1)/(hc-1), x1], [(y2-y1)/(Wc-1), (y3-y1)/(hc-1), y1]]
 * in float64 without FMA (csrc/crop.cuh: one definition for both entry points; oracle/crop.py).  BR is not used.
 *
 * ctpn_line_crop_widths_host: Wc of each of n HOST lines [n][9] -> widths[n].  CTPN_ERR_INVALID naming the line when a
 *   width is not finite or exceeds 2^20.
 * ctpn_line_crops_u8: the crops of a batch's lines, bit-identical to that warpAffine.  canvas: DEVICE uint8, image b's
 *   (h, w) = im_hw[2b..2b+1] pixels (BGR) at canvas + b * batch_pitch + y * row_pitch + 3x.  lines: DEVICE float64
 *   [batch][rows][9] (ctpn_text_lines' layout); image b's first num_lines[b] rows are cropped into out[b], a DEVICE uint8
 *   [num_lines[b]][hc][max_width[b]][3]: columns at and past a line's Wc are written as 0.  max_width[b] must be at least
 *   every Wc of the image (ctpn_line_crop_widths_host on the same lines); a line whose Wc the kernel finds larger, or not
 *   finite, gets no pixels and sets status[b] (DEVICE, or host memory the device can write) to 1 -- status is written
 *   for such images only, so one buffer can collect several launches.  Taps are clamped to the image, so no line value,
 *   NaN included, makes the kernel read outside it.  im_hw, num_lines, max_width and out are HOST arrays (1 <= batch <=
 *   64), validated before any CUDA call (CTPN_ERR_INVALID naming the image): hc range, 0 <= num_lines[b] <= rows, h, w
 *   >= 1, 3w <= row_pitch and h * row_pitch <= batch_pitch, and where num_lines[b] > 0 a non-NULL out[b] and
 *   2 <= max_width[b] <= 2^20, non-NULL canvas, lines and status.  Stream-ordered, no allocation, no synchronisation;
 *   CTPN_ERR_NO_DEVICE without a GPU.
 *
 * Source crops: the same recipe applied to the SOURCE line of each line and the source image, at full resolution.  With
 * f[b] the resize_im factor of image b, the source line is the line's corners divided by f[b], one IEEE float64 division
 * each (src = line / f, as draw_boxes divides; numpy's lines[:, :8] / f on the host gives the same bits, and
 * ctpn_line_crop_widths_host on those gives the widths), and the crop is cv2.warpAffine(source_bgr, Minv(src), ...).
 * ctpn_line_crops_strided_u8: the sources are read in place, as ctpn_resize_linear_u8_strided reads them (src, src_bytes,
 *   src_offset, src_strides, src_hw: its descriptors and its rules; a host image uploaded whole is the descriptor
 *   (w * 3, 3, 1)).  At most 64 images, one launch.
 * ctpn_line_crops_yuv420_u8: the sources are YUV 4:2:0 frames, described and checked as ctpn_resize_linear_u8_yuv420
 *   describes them; each sample is converted as cv2.cvtColor(COLOR_YUV2BGR_*) converts it.  At most 64 frames, launched
 *   in chunks of 32 (three planes' descriptors per frame).
 * Both: lines DEVICE float64 [batch][rows][9] in the resize_im frame; num_lines, max_width, out and status as for
 *   ctpn_line_crops_u8, with max_width[b] at least every source width of image b.  f, num_lines, max_width, out and the
 *   descriptors are HOST arrays (1 <= batch <= 64), validated before any CUDA call (CTPN_ERR_INVALID naming the image, and
 *   the plane): the hc range, 0 <= num_lines[b] <= rows, f[b] finite and > 0, the descriptor rules, where num_lines[b] > 0
 *   a non-NULL out[b] and 2 <= max_width[b] <= 2^20, and non-NULL lines and status when any image has lines.  Taps are
 *   clamped to the source image.  Stream-ordered, no allocation, no synchronisation; CTPN_ERR_NO_DEVICE without a GPU. */
int ctpn_line_crop_widths_host(const double *lines, int n, int hc, int *widths);
int ctpn_line_crops_u8(const void *canvas, long long batch_pitch, int row_pitch, const int *im_hw, const double *lines,
                       int batch, int rows, int hc, const int *num_lines, const int *max_width, void *const *out, int *status,
                       void *stream);
int ctpn_line_crops_strided_u8(const void *const *src, const size_t *src_bytes, const long long *src_offset,
                               const long long *src_strides, const int *src_hw, const double *f, const double *lines, int batch,
                               int rows, int hc, const int *num_lines, const int *max_width, void *const *out, int *status,
                               void *stream);
int ctpn_line_crops_yuv420_u8(const void *const *planes, const size_t *plane_bytes, const long long *plane_offset,
                              const long long *plane_strides, const int *src_hw, const double *f, const double *lines, int batch,
                              int rows, int hc, const int *num_lines, const int *max_width, void *const *out, int *status,
                              void *stream);

/* ---- RPN training targets (host; SURVEY.md 8(f) rank 4) -------------------------------------------------------------
 * The reference computes these on the CPU once per training image; so does this library (plain C++, no device work).
 * ctpn_bbox_overlaps_host: lib/utils/bbox.pyx:15-55 -- IoU with the +1 pixel convention of boxes [n][boxes_stride>=4]
 * against query_boxes [k][query_stride>=4] (x1,y1,x2,y2 in the first four columns), float64, overlaps [n][k]; 0 where
 * disjoint.  ctpn_bbox_intersections_host: bbox.pyx:57-95 -- intersection / area(query box). */
int ctpn_bbox_overlaps_host(const double *boxes, int n, int boxes_stride, const double *query_boxes, int k, int query_stride,
                            double *overlaps);
int ctpn_bbox_intersections_host(const double *boxes, int n, int boxes_stride, const double *query_boxes, int k,
                                 int query_stride, double *intersections);
/* anchor_target_layer_tf.py:78-175 and :201 fused: labels (1 fg, 0 bg, -1 ignored; BEFORE the random sub-sampling of
 * :181-198, which the caller does so that the random stream stays its own) and float32 regression targets
 * (bbox_transform.py:10-29 against each anchor's best ground truth) for all feat_h*feat_w*10 anchors in (row, col, anchor)
 * order; anchors outside the im_w x im_h image get label -1 and zero targets (_unmap, :256-267).
 * gt_boxes [num_gt][4] float64 (num_gt >= 1); gt_is_f32 != 0 when the caller's annotations were float32 (numpy then
 * keeps the ground-truth side of bbox_transform in float32); gt_ishard [num_gt] or NULL; dontcare_areas
 * [num_dontcare][4] or NULL.  cfg5 = (RPN_NEGATIVE_OVERLAP, RPN_POSITIVE_OVERLAP, RPN_CLOBBER_POSITIVES,
 * DONTCARE_AREA_INTERSECTION_HI, PRECLUDE_HARD_SAMPLES), lib/fast_rcnn/config.py:112-121. */
int ctpn_anchor_targets_host(const double *gt_boxes, int num_gt, int gt_is_f32, const unsigned char *gt_ishard,
                             const double *dontcare_areas, int num_dontcare, int feat_h, int feat_w, int feat_stride,
                             double im_h, double im_w, const double *cfg5, float *labels, float *bbox_targets);

#ifdef __cplusplus
}
#endif
#endif /* CTPN_B200_H_ */
