// Batched text-line connector on the device: TextDetector.detect for every image of a batch, reading the proposal
// layer's rois where they lie (SURVEY.md §8 f rank 3).  One CTA per image runs the stages of ctpn_text_lines_host
// (textline.cu) with the SAME per-element functions (textline.cuh), so every line equals the host connector's as float64
// bits; this object is compiled with -fmad=false (csrc/Makefile) so that no a * b + c is contracted into an FMA.
//
//   load      boxes = float32(double(roi[1:5]) / im_scale), score filter, rank (score desc, index asc) by counting
//   NMS       upper-triangle bitmask of the suppression test, then the greedy scan in 64-row blocks (as nms.cu)
//   graph     column table of the survivors by int(x1) (counting sort, ascending within a column), one thread per
//             proposal for successor / precursors
//   lines     one thread per chain head walks and fits its chain; a block scan compacts the kept lines in head order
//
// Every per-image array lives in the workspace; shared memory holds the greedy scan's suppression words (rows / 64) and
// the scan scratch only, so rows is limited by kTextMaxRows and the workspace, not by shared memory.
#include <algorithm>

#include "common.cuh"
#include "textline.cuh"

namespace ctpn {
namespace {

typedef unsigned long long u64;
constexpr int kThreads = 512;
constexpr int kTextMaxBatch = 64;
constexpr int kTextMaxRows = 1 << 16;   // 1024 suppression words = 8 KiB of shared memory

// per-image host descriptors, passed by value
struct TextBatch {
  int im_h[kTextMaxBatch], im_w[kTextMaxBatch];
  double im_scale[kTextMaxBatch];
};

// Workspace slice of one image (all offsets 256-byte aligned)
struct Slice {
  size_t box, area, score, mask, tp, sc, next, has_in, col_idx, col_start, col_fill, keep, total;
};

__host__ __device__ inline size_t al(size_t v) { return (v + 255) / 256 * 256; }

__host__ __device__ inline Slice slice_layout(int rows, int max_im_w) {
  const size_t r = (size_t)rows, words = (size_t)((rows + 63) / 64);
  Slice s;
  size_t o = 0;
  s.box = o;       o += al(r * sizeof(tl::Box));        // candidates in score order
  s.area = o;      o += al(r * sizeof(float));
  s.score = o;     o += al(r * sizeof(float));
  s.mask = o;      o += al(r * words * sizeof(u64));    // NMS suppression bits, row i: candidates j > i
  s.tp = o;        o += al(r * sizeof(tl::Box));        // NMS survivors in visiting order
  s.sc = o;        o += al(r * sizeof(float));
  s.next = o;      o += al(r * sizeof(int));
  s.has_in = o;    o += al(r * sizeof(int));
  s.col_idx = o;   o += al(r * sizeof(int));
  s.col_start = o; o += al(((size_t)max_im_w + 1) * sizeof(int));
  s.col_fill = o;  o += al((size_t)max_im_w * sizeof(int));
  s.keep = o;      o += al(r * sizeof(int));            // sorted positions of the survivors
  s.total = o;
  return s;
}

// exclusive prefix sum of v over the block; *total receives the block sum.  Every thread must call it.
__device__ int block_exclusive_scan(int v, int *total) {
  __shared__ int warp_sum[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) warp_sum[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = lane < kThreads / 32 ? warp_sum[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w += y;
    }
    if (lane < kThreads / 32) warp_sum[lane] = w;
  }
  __syncthreads();
  const int before = (warp ? warp_sum[warp - 1] : 0) + x - v;
  *total = warp_sum[kThreads / 32 - 1];
  __syncthreads();   // warp_sum is reused by the next call
  return before;
}

__global__ void __launch_bounds__(kThreads)
text_lines_kernel(const float *__restrict__ rois, const int *__restrict__ counts, int rows, const TextBatch p,
                  int oriented, tl::TextCfg cfg, int max_im_w, double *__restrict__ lines_out, int *__restrict__ num_lines,
                  int *__restrict__ status, unsigned char *__restrict__ ws) {
  extern __shared__ u64 remv[];                      // suppression words of the greedy scan, (rows + 63) / 64
  __shared__ u64 diag[64];
  __shared__ u64 s_kept;
  __shared__ int s_rows[64];
  __shared__ int s_m0, s_m, s_bad;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int im_h = p.im_h[b], im_w = p.im_w[b];
  const double im_scale = p.im_scale[b];
  const Slice L = slice_layout(rows, max_im_w);
  unsigned char *base = ws + (size_t)b * L.total;
  tl::Box *box = (tl::Box *)(base + L.box);
  float *area = (float *)(base + L.area), *score = (float *)(base + L.score);
  u64 *mask = (u64 *)(base + L.mask);
  tl::Box *tp = (tl::Box *)(base + L.tp);
  float *sc = (float *)(base + L.sc);
  int *next = (int *)(base + L.next), *has_in = (int *)(base + L.has_in), *col_idx = (int *)(base + L.col_idx);
  int *col_start = (int *)(base + L.col_start), *col_fill = (int *)(base + L.col_fill), *keep = (int *)(base + L.keep);
  const float *r = rois + (size_t)b * rows * 5;
  const int n = counts[b];
  if (n < 0 || n > rows) {                           // not a proposal-layer count for this buffer
    if (tid == 0) {
      num_lines[b] = 0;
      status[b] = 2;
    }
    return;
  }
  // ---- score filter and stable rank: position = #{passing j: s_j > s_i, or s_j == s_i and j < i} ----
  if (tid == 0) s_m0 = 0;
  __syncthreads();
  {
    int cnt = 0;
    for (int i = tid; i < n; i += kThreads) cnt += r[(size_t)i * 5] > cfg.min_score;
    if (cnt) atomicAdd(&s_m0, cnt);
  }
  for (int i = tid; i < n; i += kThreads) {
    const float s = r[(size_t)i * 5];
    if (!(s > cfg.min_score)) continue;
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      const float t = r[(size_t)j * 5];
      rank += (t > cfg.min_score) && (t > s || (t == s && j < i));
    }
    const float *q = r + (size_t)i * 5;
    const tl::Box bx{tl::blob_to_image(q[1], im_scale), tl::blob_to_image(q[2], im_scale), tl::blob_to_image(q[3], im_scale),
                     tl::blob_to_image(q[4], im_scale)};
    box[rank] = bx;
    area[rank] = tl::area_plus1(bx);
    score[rank] = s;
  }
  __syncthreads();
  const int m0 = s_m0, words = (m0 + 63) / 64;
  // ---- NMS: mask[i][w] bit t = candidate 64 w + t (> i) is suppressed by i ----
  for (long long task = tid; task < (long long)m0 * words; task += kThreads) {
    const int i = (int)(task / words), w = (int)(task % words);
    if (w < i / 64) continue;                        // never read: the scan only ORs words of later blocks
    const tl::Box me = box[i];
    const float a = area[i];
    u64 bits = 0;
    const int j0 = 64 * w, j1 = min(j0 + 64, m0);
    for (int j = max(j0, i + 1); j < j1; ++j)
      if (tl::nms_suppresses(me, a, box[j], area[j], cfg.nms_thresh)) bits |= 1ull << (j - j0);
    mask[(size_t)i * words + w] = bits;
  }
  for (int w = tid; w < words; w += kThreads) remv[w] = 0;
  if (tid == 0) s_m = 0;
  __syncthreads();
  // greedy scan: thread 0 resolves a block from its diagonal words, all threads OR the kept rows into later blocks
  for (int blk = 0; blk < words; ++blk) {
    const int base_row = blk * 64;
    if (tid < 64) diag[tid] = base_row + tid < m0 ? mask[(size_t)(base_row + tid) * words + blk] : 0ull;
    __syncthreads();
    if (tid == 0) {
      u64 cur = remv[blk], kept = 0;
      int nk = s_m;
      const int lim = min(64, m0 - base_row);
      for (int t = 0; t < lim; ++t)
        if (!((cur >> t) & 1ull)) {
          s_rows[__popcll(kept)] = t;
          kept |= 1ull << t;
          keep[nk++] = base_row + t;
          cur |= diag[t];
        }
      s_kept = kept;
      s_m = nk;
    }
    __syncthreads();
    const u64 kept = s_kept;
    const int cnt = __popcll(kept);
    for (int w = blk + 1 + tid; w < words; w += kThreads) {
      u64 acc = remv[w];
      for (int q = 0; q < cnt; ++q) acc |= mask[(size_t)(base_row + s_rows[q]) * words + w];
      remv[w] = acc;
    }
    __syncthreads();
  }
  const int m = s_m;
  // ---- survivors in visiting order; the column table's range check (the host raises IndexError there) ----
  if (tid == 0) s_bad = 0;
  __syncthreads();
  for (int k = tid; k < m; k += kThreads) {
    const tl::Box bx = box[keep[k]];
    tp[k] = bx;
    sc[k] = score[keep[k]];
    next[k] = -1;
    has_in[k] = 0;
    if (!tl::column_ok(bx.x1, im_w)) s_bad = 1;
  }
  for (int c = tid; c <= im_w; c += kThreads) col_start[c] = 0;
  __syncthreads();
  if (s_bad) {
    if (tid == 0) {
      num_lines[b] = 0;
      status[b] = 1;
    }
    return;
  }
  // ---- column table: counts, exclusive scan, fill, ascending order within each column ----
  for (int k = tid; k < m; k += kThreads) atomicAdd(&col_start[(int)tp[k].x1 + 1], 1);
  __syncthreads();
  int carry = 0;
  for (int c0 = 0; c0 < im_w; c0 += kThreads) {
    const int c = c0 + tid;
    const int v = c < im_w ? col_start[c + 1] : 0;
    int total;
    const int before = block_exclusive_scan(v, &total);
    if (c < im_w) {
      col_start[c + 1] = carry + before + v;
      col_fill[c] = carry + before;
    }
    carry += total;
  }
  __syncthreads();
  for (int k = tid; k < m; k += kThreads) col_idx[atomicAdd(&col_fill[(int)tp[k].x1], 1)] = k;
  __syncthreads();
  for (int c = tid; c < im_w; c += kThreads) {       // insertion sort: a column holds a handful of proposals
    const int lo = col_start[c], hi = col_start[c + 1];
    for (int a = lo + 1; a < hi; ++a) {
      const int v = col_idx[a];
      int q = a - 1;
      while (q >= lo && col_idx[q] > v) {
        col_idx[q + 1] = col_idx[q];
        --q;
      }
      col_idx[q + 1] = v;
    }
  }
  __syncthreads();
  // ---- graph ----
  for (int i = tid; i < m; i += kThreads) {
    const int s = tl::successor(i, tp, sc, col_start, col_idx, im_w, cfg);
    if (s >= 0) {
      next[i] = s;
      has_in[s] = 1;
    }
  }
  __syncthreads();
  // ---- one thread per chain head; kept lines compacted in ascending head order ----
  double *out = lines_out + (size_t)b * rows * 9;
  int written = 0;
  for (int i0 = 0; i0 < m; i0 += kThreads) {
    const int i = i0 + tid;
    double line[9];
    bool ok = false;
    if (i < m && !has_in[i] && next[i] >= 0) {
      const tl::Chain chain{tp, sc, next, i, tl::chain_length(next, i, m)};
      ok = tl::chain_line(chain, im_h, im_w, oriented, cfg, line);
    }
    int total;
    const int pos = written + block_exclusive_scan(ok ? 1 : 0, &total);
    if (ok)
      for (int q = 0; q < 9; ++q) out[(size_t)pos * 9 + q] = line[q];
    written += total;
  }
  if (tid == 0) {
    num_lines[b] = written;
    status[b] = 0;
  }
}

}  // namespace
}  // namespace ctpn

using namespace ctpn;

extern "C" size_t ctpn_text_lines_workspace_bytes(int batch, int rows, int max_im_w) {
  if (batch <= 0 || rows < 0 || max_im_w <= 0) return 0;
  return (size_t)batch * slice_layout(rows, max_im_w).total;
}

extern "C" int ctpn_text_lines(const float *rois, const int *counts, int batch, int rows, const int *im_hw, const double *im_scale,
                               int oriented, const float *cfg9, double *lines_out, int *num_lines, int *status, void *ws,
                               size_t ws_bytes, void *stream) {
  CTPN_REQUIRE(rois && counts && im_hw && im_scale && lines_out && num_lines && status && ws, "ctpn_text_lines: null pointer");
  CTPN_REQUIRE(batch >= 1 && batch <= kTextMaxBatch, "ctpn_text_lines: batch = %d, must be 1..%d", batch, kTextMaxBatch);
  CTPN_REQUIRE(rows >= 0 && rows <= kTextMaxRows, "ctpn_text_lines: rows = %d, must be 0..%d", rows, kTextMaxRows);
  CTPN_REQUIRE(oriented == 0 || oriented == 1, "ctpn_text_lines: oriented = %d, must be 0 or 1", oriented);
  TextBatch p;
  int max_w = 1;
  for (int b = 0; b < batch; ++b) {
    const int h = im_hw[2 * b], w = im_hw[2 * b + 1];
    const double s = im_scale[b];
    CTPN_REQUIRE(h > 0 && w > 0, "ctpn_text_lines: image %d: bad size %d x %d", b, h, w);
    CTPN_REQUIRE(s > 0.0 && s <= 1e30, "ctpn_text_lines: image %d: im_scale %g must be > 0 and finite", b, s);
    p.im_h[b] = h;
    p.im_w[b] = w;
    p.im_scale[b] = s;
    max_w = std::max(max_w, w);
  }
  const size_t need = ctpn_text_lines_workspace_bytes(batch, rows, max_w);
  if (ws_bytes < need) {
    set_error("ctpn_text_lines: workspace %zu < %zu bytes", ws_bytes, need);
    return CTPN_ERR_INVALID;
  }
  const tl::TextCfg cfg = tl::parse_cfg(cfg9);
  int sms = 0;
  if (int rc = current_sm_count(&sms)) return rc;    // also CTPN_ERR_NO_DEVICE without a GPU
  const size_t smem = (size_t)((rows + 63) / 64) * sizeof(u64);
  ProfScope prof("text_lines", 0.0, (cudaStream_t)stream);
  text_lines_kernel<<<batch, kThreads, smem, (cudaStream_t)stream>>>(rois, counts, rows, p, oriented, cfg, max_w, lines_out,
                                                                     num_lines, status, (unsigned char *)ws);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}
