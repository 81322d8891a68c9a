// RPN proposal layer on the device, batched over images:
//   decode (fg score, anchor synthesis, vertical bbox decode, clip, min-size filter)
//   -> stable segmented radix sort by score (descending; ties by ascending anchor index)
//   -> top pre_nms_topN -> bitmask NMS with on-device greedy scan (early exit at post_nms_topN)
//   -> rois [score, x1, y1, x2, y2].
// Replaces lib/rpn_msr/proposal_layer_tf.py:14-157 (host numpy inside tf.py_func) and the
// host<->device round trips of lib/utils/nms_kernel.cu:91-144.
//
// Exactness: all box arithmetic is float32 in the reference's operation order with no FMA
// contraction; exp() is evaluated in double and rounded once (== oracle exp_mode='rounded').
#include "common.cuh"
#include "nms_iou.cuh"

namespace ctpn {

typedef unsigned long long u64;

int nms_sorted_launch(const float *boxes, const int *counts, int batch, int max_n, float thresh,
                      int max_keep, int keep_stride, int *keep_out, int *num_out, void *workspace,
                      size_t workspace_bytes, cudaStream_t st, const int *gate);

// generate_anchors.py:26 heights -> (y1, y2) of the 10 base anchors; x is always [0, 15].
__constant__ int c_anchor_y[2][10][2] = {
    {{2, 13}, {0, 15}, {-4, 19}, {-9, 24}, {-16, 31}, {-26, 41}, {-41, 56}, {-62, 77}, {-91, 106}, {-134, 149}},  // py3
    {{2, 12}, {0, 15}, {-3, 18}, {-8, 23}, {-16, 31}, {-26, 41}, {-40, 55}, {-61, 76}, {-91, 106}, {-133, 148}}   // py2
};

__device__ __forceinline__ uint32_t desc_key(float s) {
  uint32_t u = __float_as_uint(s == 0.f ? 0.f : s);   // -0 ties with +0 (then ascending index), as in the oracle's sort
  uint32_t asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ~asc;   // ascending key order == descending score
}

__global__ void __launch_bounds__(256)
proposal_decode_kernel(const float *__restrict__ cls, int cls_is_logit, const float *__restrict__ bbox,
                       const float *__restrict__ im_info, int H, int W, int feat_stride, float min_size,
                       int py2, float nms_thresh, float4 *__restrict__ boxes, float *__restrict__ scores,
                       uint32_t *__restrict__ keys, uint8_t *__restrict__ valid, int *__restrict__ unstructured,
                       const int *__restrict__ feat_hw) {
  const int NA = H * W * 10;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int img = blockIdx.y;
  if (i >= NA) return;
  const int a = i % 10;
  const int cell = i / 10;
  const int w = cell % W, h = cell / W;
  const size_t off = (size_t)img * NA + i;
  if (feat_hw && (h >= feat_hw[2 * img] || w >= feat_hw[2 * img + 1])) {   // ragged batch: a cell outside the image's map
    boxes[off] = make_float4(0.f, 0.f, 0.f, 0.f);
    scores[off] = 0.f;
    keys[off] = desc_key(0.f);
    valid[off] = 0;
    return;
  }
  // fg score: channel 2a+1 of the pair (proposal_layer_tf.py:65)
  const float *cp = cls + ((size_t)img * H * W + cell) * 20 + 2 * a;
  float score;
  if (cls_is_logit) {   // spatial_softmax over the (bg, fg) pair, network.py:332-337
    float l0 = cp[0], l1 = cp[1];
    float m = fmaxf(l0, l1);
    float e0 = expf(__fsub_rn(l0, m)), e1 = expf(__fsub_rn(l1, m));
    score = __fdiv_rn(e1, __fadd_rn(e0, e1));
  } else {
    score = cp[1];
  }
  const float *dp = bbox + ((size_t)img * H * W + cell) * 40 + 4 * a;
  const float dy = dp[1], dh = dp[3];
  // anchor (proposal_layer_tf.py:83-99), integer valued
  const float ax1 = (float)(w * feat_stride), ax2 = (float)(w * feat_stride + 15);
  const float ay1 = (float)(h * feat_stride + c_anchor_y[py2][a][0]);
  const float ay2 = (float)(h * feat_stride + c_anchor_y[py2][a][1]);
  // bbox_transform_inv (bbox_transform.py:36-65): dx, dw ignored
  const float widths = __fadd_rn(__fsub_rn(ax2, ax1), 1.0f);
  const float heights = __fadd_rn(__fsub_rn(ay2, ay1), 1.0f);
  const float ctr_x = __fadd_rn(ax1, __fmul_rn(0.5f, widths));
  const float ctr_y = __fadd_rn(ay1, __fmul_rn(0.5f, heights));
  const float pcy = __fadd_rn(__fmul_rn(dy, heights), ctr_y);
  const float ph = __fmul_rn((float)exp((double)dh), heights);
  float x1 = __fsub_rn(ctr_x, __fmul_rn(0.5f, widths));
  float y1 = __fsub_rn(pcy, __fmul_rn(0.5f, ph));
  float x2 = __fadd_rn(ctr_x, __fmul_rn(0.5f, widths));
  float y2 = __fadd_rn(pcy, __fmul_rn(0.5f, ph));
  // clip_boxes (bbox_transform.py:67-80)
  const float *info = im_info + img * 3;
  const float hx = __fsub_rn(info[1], 1.0f), hy = __fsub_rn(info[0], 1.0f);
  x1 = fmaxf(fminf(x1, hx), 0.f);
  y1 = fmaxf(fminf(y1, hy), 0.f);
  x2 = fmaxf(fminf(x2, hx), 0.f);
  y2 = fmaxf(fminf(y2, hy), 0.f);
  // _filter_boxes (proposal_layer_tf.py:160-165) with min_size * im_info[2]
  const float ms = __fmul_rn(min_size, info[2]);
  const float ws = __fadd_rn(__fsub_rn(x2, x1), 1.0f), hs = __fadd_rn(__fsub_rn(y2, y1), 1.0f);
  boxes[off] = make_float4(x1, y1, x2, y2);
  scores[off] = score;
  keys[off] = desc_key(score);
  const bool ok = ws >= ms && hs >= ms;
  valid[off] = ok ? 1 : 0;
  // Column structure check for the fast NMS path: a kept box must start exactly at its anchor column,
  // end within it (<= 1 px shared with the next column) and be wide enough that a 1-px overlap can
  // never reach the NMS threshold: IoU <= 1 / (w + w' - 1) <= 1 / (2 w_min - 1) < thresh.
  if (ok && unstructured && (x1 != ax1 || x2 > ax1 + (float)feat_stride || (2.f * ws - 1.f) * nms_thresh <= 1.f))
    unstructured[img] = 1;
}

// ---- segmented stable LSD radix sort: one CTA per image, 4 passes of 8 bits ---------------
constexpr int kSortThreads = 1024;
constexpr int kSortWarps = kSortThreads / 32;
constexpr size_t kSortSmem = (512 + 2 * kSortWarps * 256) * sizeof(int);

__global__ void __launch_bounds__(kSortThreads)
proposal_sort_kernel(const uint32_t *__restrict__ keys, const uint8_t *__restrict__ valid,
                     const float4 *__restrict__ boxes, int NA, int max_n, uint2 *__restrict__ buf_a,
                     uint2 *__restrict__ buf_b, float4 *__restrict__ sorted_boxes,
                     int *__restrict__ sorted_idx, int *__restrict__ counts, int W_cols, int *__restrict__ col_start) {
  extern __shared__ int sort_smem[];
  int *hist = sort_smem;                   // [256]
  int *base = hist + 256;                  // [256]
  int *wc = base + 256;                    // [warps][256] per-warp digit counts of the current tile
  int *wo = wc + kSortWarps * 256;         // [warps][256] per-warp output offsets of the current tile
  __shared__ int s_total;
  const int img = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t *k0 = keys + (size_t)img * NA;
  const uint8_t *v0 = valid + (size_t)img * NA;
  uint2 *bufs[2] = {buf_a + (size_t)img * NA, buf_b + (size_t)img * NA};
  for (int k = tid; k < kSortWarps * 256; k += kSortThreads) wc[k] = 0;
  int n_in = NA;
  // passes 0-3: the 32-bit score key.  Optional pass 4 (W_cols > 0): the top max_n entries, stably re-bucketed by
  // feature-map column (payload = position in the score order) for the column-wise NMS -- each column's candidates
  // end up contiguous and still in score order, so the NMS CTAs do not have to scan the whole list.
  const int npass = W_cols > 0 ? 5 : 4;
  for (int pass = 0; pass < npass; ++pass) {
    const int shift = 8 * pass;
    const uint2 *src = bufs[(pass + 1) & 1];   // pass 0 reads keys/valid instead
    uint2 *dst = bufs[pass & 1];
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < n_in; i += kSortThreads) {
      bool has;
      uint32_t key;
      if (pass == 0) { has = v0[i] != 0; key = k0[i]; } else { has = true; key = src[i].x; }
      if (pass == 4) atomicAdd(&hist[(src[i].y / 10u) % (uint32_t)W_cols], 1);
      else if (has) atomicAdd(&hist[(key >> shift) & 255], 1);
    }
    __syncthreads();
    if (warp == 0) {   // exclusive scan of 256 bins: 8 per lane
      int loc[8], sum = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) { loc[k] = hist[lane * 8 + k]; sum += loc[k]; }
      int incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      int run = incl - sum;
#pragma unroll
      for (int k = 0; k < 8; ++k) { base[lane * 8 + k] = run; run += loc[k]; }
    }
    __syncthreads();
    if (pass == 4 && tid <= W_cols) col_start[img * 257 + tid] = tid < 256 ? base[tid] : n_in;
    if (pass == 4) __syncthreads();
    for (int start = 0; start < n_in; start += kSortThreads) {
      const int i = start + tid;
      bool has = i < n_in;
      uint32_t key = 0, idx = 0;
      if (has) {
        if (pass == 0) { has = v0[i] != 0; key = k0[i]; idx = (uint32_t)i; }
        else { uint2 p = src[i]; key = p.x; idx = p.y; }
      }
      const uint32_t d = !has ? 0x1FFu : pass == 4 ? (idx / 10u) % (uint32_t)W_cols : ((key >> shift) & 255u);
      const uint32_t peers = __match_any_sync(0xffffffffu, d);
      const int rank = __popc(peers & ((1u << lane) - 1u));
      if (has && rank == 0) wc[warp * 256 + d] = __popc(peers);
      __syncthreads();
      if (tid < 256) {
        int run = base[tid];
#pragma unroll 8
        for (int w = 0; w < kSortWarps; ++w) {
          int c = wc[w * 256 + tid];
          wo[w * 256 + tid] = run;
          wc[w * 256 + tid] = 0;
          run += c;
        }
        base[tid] = run;
      }
      __syncthreads();
      if (has) dst[wo[warp * 256 + d] + rank] = make_uint2(pass == 4 ? (uint32_t)i : key, idx);
    }
    __syncthreads();
    if (pass == 0) {   // number of valid candidates = total of the first histogram
      if (tid == 0) { int t = 0; for (int k = 0; k < 256; ++k) t += hist[k]; s_total = t; }
      __syncthreads();
      n_in = s_total;
    }
    if (pass == 3) n_in = min(n_in, max_n);   // only the top max_n take part in the column pass
  }
  // after 4 passes the result sits in bufs[1]; keep the top max_n and gather their boxes
  const uint2 *res = bufs[1];
  const int n_out = min(n_in, max_n);
  for (int r = tid; r < n_out; r += kSortThreads) {
    int idx = (int)res[r].y;
    sorted_boxes[(size_t)img * max_n + r] = boxes[(size_t)img * NA + idx];
    sorted_idx[(size_t)img * max_n + r] = idx;
  }
  if (tid == 0) counts[img] = n_out;
}

__global__ void proposal_emit_kernel(const float4 *__restrict__ sorted_boxes, const int *__restrict__ sorted_idx,
                                     const float *__restrict__ scores, const int *__restrict__ keep,
                                     const int *__restrict__ num, int NA, int max_n, int post, int kstride,
                                     float *__restrict__ rois, int *__restrict__ index_out,
                                     int *__restrict__ count_out, int W, const int *__restrict__ feat_hw) {
  const int img = blockIdx.y;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= post) return;
  const int n = min(num[img], post);
  float *r = rois + ((size_t)img * post + k) * 5;
  if (k < n) {
    int pos = keep[(size_t)img * kstride + k];
    int idx = sorted_idx[(size_t)img * max_n + pos];
    float4 b = sorted_boxes[(size_t)img * max_n + pos];
    r[0] = scores[(size_t)img * NA + idx];
    r[1] = b.x; r[2] = b.y; r[3] = b.z; r[4] = b.w;
    if (index_out) {
      int out_idx = idx;
      if (feat_hw) {     // image-local (h * fw + w) * 10 + a: monotone in the canvas index, so the tie order is the same
        const int cell = idx / 10;
        out_idx = ((cell / W) * feat_hw[2 * img + 1] + cell % W) * 10 + idx % 10;
      }
      index_out[(size_t)img * post + k] = out_idx;
    }
  } else {
    r[0] = r[1] = r[2] = r[3] = r[4] = 0.f;
    if (index_out) index_out[(size_t)img * post + k] = -1;
  }
  if (k == 0) count_out[img] = n;
}

// ---- column-wise NMS ---------------------------------------------------------------------------
// CTPN proposals of different feature-map columns overlap by at most one pixel column, so greedy NMS
// over the score-sorted list decomposes EXACTLY into independent per-column problems of <= H*10 boxes
// (SURVEY.md App. A.4; the decode kernel verifies the precondition per image and the generic bitmask
// path takes over when it does not hold).  One CTA per (column, image): ordered gather of the
// column's boxes from the sorted list, pairwise mask in shared memory, warp-serial greedy scan.
constexpr int kColThreads = 256;

__global__ void __launch_bounds__(kColThreads)
proposal_column_nms_kernel(const float4 *__restrict__ sorted_boxes, const int *__restrict__ sorted_idx,
                           const int *__restrict__ counts, const int *__restrict__ unstructured, int max_n, int H,
                           int W, float thresh, uint8_t *__restrict__ kept_flags, const uint2 *__restrict__ colbuf,
                           const int *__restrict__ col_start, int NA) {
  const int col = blockIdx.x, img = blockIdx.y;
  if (unstructured[img]) return;
  const int cap = H * 10, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  extern __shared__ __align__(16) unsigned char col_smem[];
  float4 *box = reinterpret_cast<float4 *>(col_smem);
  u64 *mask = reinterpret_cast<u64 *>(box + cap);
  const int wc_max = (cap + 63) / 64;
  float *area = reinterpret_cast<float *>(mask + (size_t)cap * wc_max);
  int *pos = reinterpret_cast<int *>(area + cap);
  __shared__ int warp_cnt[kColThreads / 32];
  const int n = counts[img];
  const float4 *sb = sorted_boxes + (size_t)img * max_n;
  const int *si = sorted_idx + (size_t)img * max_n;
  int total = 0;
  if (col_start) {   // the sort kernel already bucketed the score-ordered list by column
    const int seg0 = col_start[img * 257 + col];
    total = col_start[img * 257 + col + 1] - seg0;
    const uint2 *cb = colbuf + (size_t)img * NA + seg0;
    for (int k = tid; k < min(total, cap); k += kColThreads) {
      const int r = (int)cb[k].x;
      pos[k] = r;
      const float4 b = sb[r];
      box[k] = b;
      area[k] = box_area(b);
    }
    __syncthreads();
  } else
  for (int base = 0; base < n; base += kColThreads) {
    const int r = base + tid;
    const bool pred = r < n && ((si[r] / 10) % W == col);
    const unsigned bal = __ballot_sync(0xffffffffu, pred);
    if (lane == 0) warp_cnt[warp] = __popc(bal);
    __syncthreads();
    int before = 0, tile = 0;
#pragma unroll
    for (int w = 0; w < kColThreads / 32; ++w) { const int c = warp_cnt[w]; tile += c; if (w < warp) before += c; }
    if (pred) {
      const int k = total + before + __popc(bal & ((1u << lane) - 1u));
      if (k < cap) { pos[k] = r; const float4 b = sb[r]; box[k] = b; area[k] = box_area(b); }
    }
    total += tile;
    __syncthreads();
  }
  const int nc = min(total, cap);
  const int wc = (nc + 63) / 64;
  for (int item = tid; item < nc * wc; item += kColThreads) {
    const int i = item / wc, wj = item % wc;
    const float4 me = box[i];
    const float sme = area[i];
    u64 bits = 0;
    const int j0 = wj * 64;
    for (int jj = max(0, i + 1 - j0); jj < 64 && j0 + jj < nc; ++jj)
      if (iou_above(me, sme, box[j0 + jj], area[j0 + jj], thresh)) bits |= 1ULL << jj;
    mask[(size_t)i * wc + wj] = bits;
  }
  __syncthreads();
  if (warp == 0) {   // lane l owns word l of the running suppression vector (wc <= 32)
    u64 remv = 0;
    uint8_t *kf = kept_flags + (size_t)img * max_n;
    for (int i = 0; i < nc; ++i) {
      const u64 word = __shfl_sync(0xffffffffu, remv, i >> 6);
      const bool keep = !((word >> (i & 63)) & 1ULL);
      if (keep && lane < wc) remv |= mask[(size_t)i * wc + lane];
      if (lane == 0) kf[pos[i]] = keep ? 1 : 0;
    }
  }
}

// first `post` kept positions of every image, in sorted (score) order
__global__ void __launch_bounds__(1024)
proposal_compact_kernel(const uint8_t *__restrict__ kept_flags, const int *__restrict__ counts,
                        const int *__restrict__ unstructured, int max_n, int post, int *__restrict__ keep,
                        int *__restrict__ num) {
  const int img = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (unstructured[img]) return;
  __shared__ int warp_cnt[32];
  const int n = counts[img];
  const uint8_t *kf = kept_flags + (size_t)img * max_n;
  int total = 0;
  for (int base = 0; base < n && total < post; base += 1024) {
    const int r = base + tid;
    const bool pred = r < n && kf[r] != 0;
    const unsigned bal = __ballot_sync(0xffffffffu, pred);
    if (lane == 0) warp_cnt[warp] = __popc(bal);
    __syncthreads();
    int before = 0, tile = 0;
#pragma unroll
    for (int w = 0; w < 32; ++w) { const int c = warp_cnt[w]; tile += c; if (w < warp) before += c; }
    if (pred) {
      const int k = total + before + __popc(bal & ((1u << lane) - 1u));
      if (k < post) keep[(size_t)img * post + k] = r;
    }
    total += tile;
    __syncthreads();
  }
  if (tid == 0) num[img] = min(total, post);
}

static size_t column_smem_bytes(int H) {
  const size_t cap = (size_t)H * 10, wc = (cap + 63) / 64;
  return cap * sizeof(float4) + cap * wc * sizeof(u64) + cap * sizeof(float) + cap * sizeof(int);
}

struct ProposalWs {
  size_t boxes, scores, keys, valid, buf_a, buf_b, sorted_boxes, sorted_idx, counts, keep, num, mask, total;
  size_t unstructured, kept_flags, col_start;
  size_t mask_bytes;
};

static ProposalWs proposal_layout(int batch, int NA, int max_n, int post) {
  ProposalWs w;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t at = o; o = align_up(o + bytes, 256); return at; };
  w.boxes = take((size_t)batch * NA * sizeof(float4));
  w.scores = take((size_t)batch * NA * sizeof(float));
  w.keys = take((size_t)batch * NA * sizeof(uint32_t));
  w.valid = take((size_t)batch * NA);
  w.buf_a = take((size_t)batch * NA * sizeof(uint2));
  w.buf_b = take((size_t)batch * NA * sizeof(uint2));
  w.sorted_boxes = take((size_t)batch * max_n * sizeof(float4));
  w.sorted_idx = take((size_t)batch * max_n * sizeof(int));
  w.counts = take((size_t)batch * sizeof(int));
  w.keep = take((size_t)batch * post * sizeof(int));
  w.num = take((size_t)batch * sizeof(int));
  w.unstructured = take((size_t)batch * sizeof(int));
  w.kept_flags = take((size_t)batch * max_n);
  w.col_start = take((size_t)batch * 257 * sizeof(int));
  w.mask_bytes = ctpn_nms_workspace_bytes(batch, max_n);
  w.mask = take(w.mask_bytes);
  w.total = o;
  return w;
}

}  // namespace ctpn

using namespace ctpn;

static inline int eff_max_n(int NA, int pre) { return (pre > 0 && pre < NA) ? pre : NA; }

extern "C" size_t ctpn_proposals_workspace_bytes(int batch, int H, int W, int pre_nms_topN) {
  if (batch <= 0 || H <= 0 || W <= 0) return 0;
  int NA = H * W * 10;
  // post_nms_topN is not known here; the keep list is sized for the worst case (max_n)
  return proposal_layout(batch, NA, eff_max_n(NA, pre_nms_topN), eff_max_n(NA, pre_nms_topN)).total;
}

static int proposals_run(const float *cls, int cls_is_logit, const float *bbox, const float *im_info, const int *feat_hw,
                         int batch, int H, int W, int feat_stride, int pre_nms_topN, int post_nms_topN, float nms_thresh,
                         float min_size, int anchors_py2, float *rois_out, int *index_out, int *count_out, void *workspace,
                         size_t workspace_bytes, void *stream) {
  CTPN_REQUIRE(cls && bbox && im_info && rois_out && count_out, "ctpn_proposals: null pointer");
  CTPN_REQUIRE(batch > 0 && H > 0 && W > 0, "ctpn_proposals: bad shape batch=%d H=%d W=%d", batch, H, W);
  CTPN_REQUIRE(batch <= 65535, "ctpn_proposals: batch too large");
  const int NA = H * W * 10;
  const int max_n = eff_max_n(NA, pre_nms_topN);
  const int post = (post_nms_topN > 0 && post_nms_topN < max_n) ? post_nms_topN : max_n;
  // rois_out rows: the caller sizes it with post_nms_topN when > 0, else with max_n
  const int out_rows = post_nms_topN > 0 ? post_nms_topN : max_n;
  ProposalWs w = proposal_layout(batch, NA, max_n, eff_max_n(NA, pre_nms_topN));
  if (workspace_bytes < w.total || !workspace) {
    set_error("ctpn_proposals: workspace %zu < %zu bytes", workspace_bytes, w.total);
    return CTPN_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  char *ws = (char *)workspace;
  float4 *boxes = (float4 *)(ws + w.boxes);
  float *scores = (float *)(ws + w.scores);
  uint32_t *keys = (uint32_t *)(ws + w.keys);
  uint8_t *valid = (uint8_t *)(ws + w.valid);
  float4 *sorted_boxes = (float4 *)(ws + w.sorted_boxes);
  int *sorted_idx = (int *)(ws + w.sorted_idx);
  int *counts = (int *)(ws + w.counts);
  int *keep = (int *)(ws + w.keep);
  int *num = (int *)(ws + w.num);
  dim3 g1(ceil_div(NA, 256), batch);
  ProfScope prof_all("proposals (decode+sort+nms+emit)", (double)batch * NA * 24.0, st);
  // column-wise NMS is possible when one column's boxes fit in shared memory and columns do not overlap
  const size_t col_smem = column_smem_bytes(H);
#ifdef CTPN_DEBUG   // test library: force the generic bitmask NMS / the un-fused column gather (read once)
  static const bool force_generic = getenv("CTPN_GENERIC_NMS") != nullptr, force_gather = getenv("CTPN_COLUMN_GATHER") != nullptr;
#else
  constexpr bool force_generic = false, force_gather = false;
#endif
  const bool try_columns = feat_stride >= 16 && col_smem <= 200 * 1024 && H * 10 <= 2048 && W <= 65535 && !force_generic;
  int *unstructured = (int *)(ws + w.unstructured);
  CTPN_CUDA(cudaMemsetAsync(unstructured, 0, (size_t)batch * sizeof(int), st));
  proposal_decode_kernel<<<g1, 256, 0, st>>>(cls, cls_is_logit, bbox, im_info, H, W, feat_stride, min_size,
                                             anchors_py2 ? 1 : 0, nms_thresh, boxes, scores, keys, valid,
                                             try_columns ? unstructured : nullptr, feat_hw);
  CTPN_LAUNCH_CHECK();
  CTPN_CUDA(cudaFuncSetAttribute(proposal_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSortSmem));
  // W <= 256: the sort kernel also buckets the survivors by column (one more 8-bit pass)
  const bool bucket = try_columns && W <= 256 && !force_gather;
  int *col_start = (int *)(ws + w.col_start);
  proposal_sort_kernel<<<batch, kSortThreads, kSortSmem, st>>>(keys, valid, boxes, NA, max_n, (uint2 *)(ws + w.buf_a),
                                                       (uint2 *)(ws + w.buf_b), sorted_boxes, sorted_idx, counts,
                                                       bucket ? W : 0, col_start);
  CTPN_LAUNCH_CHECK();
  if (try_columns) {
    uint8_t *kept_flags = (uint8_t *)(ws + w.kept_flags);
    if (col_smem > 48 * 1024)
      CTPN_CUDA(cudaFuncSetAttribute(proposal_column_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)col_smem));
    proposal_column_nms_kernel<<<dim3(W, batch), kColThreads, col_smem, st>>>(sorted_boxes, sorted_idx, counts, unstructured,
                                                                           max_n, H, W, nms_thresh, kept_flags,
                                                                           (const uint2 *)(ws + w.buf_a), bucket ? col_start : nullptr, NA);
    CTPN_LAUNCH_CHECK();
    proposal_compact_kernel<<<batch, 1024, 0, st>>>(kept_flags, counts, unstructured, max_n, post, keep, num);
    CTPN_LAUNCH_CHECK();
  }
  // generic bitmask NMS: every image when the column path is off, else only images flagged unstructured
  int rc = nms_sorted_launch((const float *)sorted_boxes, counts, batch, max_n, nms_thresh, post, post, keep, num,
                             ws + w.mask, w.mask_bytes, st, try_columns ? unstructured : nullptr);
  if (rc) return rc;
  dim3 g3(ceil_div(out_rows, 128), batch);
  proposal_emit_kernel<<<g3, 128, 0, st>>>(sorted_boxes, sorted_idx, scores, keep, num, NA, max_n, out_rows, post, rois_out,
                                           index_out, count_out, W, feat_hw);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

extern "C" int ctpn_proposals(const float *cls, int cls_is_logit, const float *bbox, const float *im_info, int batch,
                              int H, int W, int feat_stride, int pre_nms_topN, int post_nms_topN, float nms_thresh,
                              float min_size, int anchors_py2, float *rois_out, int *index_out, int *count_out,
                              void *workspace, size_t workspace_bytes, void *stream) {
  return proposals_run(cls, cls_is_logit, bbox, im_info, nullptr, batch, H, W, feat_stride, pre_nms_topN, post_nms_topN,
                       nms_thresh, min_size, anchors_py2, rois_out, index_out, count_out, workspace, workspace_bytes, stream);
}

extern "C" int ctpn_proposals_ragged(const float *cls, int cls_is_logit, const float *bbox, const float *im_info,
                                     const int *feat_hw, int batch, int H, int W, int feat_stride, int pre_nms_topN,
                                     int post_nms_topN, float nms_thresh, float min_size, int anchors_py2, float *rois_out,
                                     int *index_out, int *count_out, void *workspace, size_t workspace_bytes, void *stream) {
  CTPN_REQUIRE(feat_hw, "ctpn_proposals_ragged: null feat_hw");
  return proposals_run(cls, cls_is_logit, bbox, im_info, feat_hw, batch, H, W, feat_stride, pre_nms_topN, post_nms_topN,
                       nms_thresh, min_size, anchors_py2, rois_out, index_out, count_out, workspace, workspace_bytes, stream);
}
