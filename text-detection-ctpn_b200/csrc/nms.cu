// Greedy NMS on the device: pairwise-IoU bitmask (upper triangle only) + an on-device greedy
// scan with early exit, batched over images.  Replaces lib/utils/nms_kernel.cu (which ships
// the full n x n/64 mask back to the host and scans it there, nms_kernel.cu:115-139).
//
// Bit-exactness contract (tests/test_nms_gpu.py): the IoU is evaluated in float32 with the
// same operation order as nms_kernel.cu:24-32 / nms_wrapper.py:30,37-44 and WITHOUT fused
// multiply-add, so keep lists equal the CPU oracle's for identical sorted input.
#include <mutex>

#include "common.cuh"
#include "nms_iou.cuh"

namespace ctpn {

typedef unsigned long long u64;
constexpr int kNmsTile = 64;

// grid G, 64 threads.  Each CTA walks, image after image, the (row block, column block) pairs of the upper triangle
// with stride G; thread = one row box against the 64 boxes of the column block.
__global__ void __launch_bounds__(kNmsTile)
nms_mask_kernel(const float4 *__restrict__ boxes, const int *__restrict__ counts, int batch, int max_n,
                int col_blocks, float thresh, u64 *__restrict__ mask, const int *__restrict__ gate) {
  __shared__ float4 cbox[kNmsTile];
  __shared__ float carea[kNmsTile];
  const int t = threadIdx.x;
  // the grid is one-dimensional and every CTA walks all images: a batch whose images all took the column-wise path (the
  // usual case inside the proposal layer) costs one gate test per image instead of a grid of empty CTAs per image
  for (int img = 0; img < batch; ++img) {
    if (gate && gate[img] == 0) continue;   // this image is handled by the column-wise path
    const int n = counts ? min(counts[img], max_n) : max_n;
    const int nb = (n + kNmsTile - 1) / kNmsTile;
    const float4 *b = boxes + (size_t)img * max_n;
    for (int pair = blockIdx.x; pair < nb * nb; pair += gridDim.x) {
      const int rb = pair / nb, cb = pair % nb;
      if (cb < rb) continue;
      const int col_size = min(n - cb * kNmsTile, kNmsTile);
      __syncthreads();
      if (t < col_size) {
        float4 v = b[cb * kNmsTile + t];
        cbox[t] = v;
        carea[t] = box_area(v);
      }
      __syncthreads();
      const int row = rb * kNmsTile + t;
      if (row < n) {
        float4 me = b[row];
        float sme = box_area(me);
        u64 bits = 0;
        int start = (rb == cb) ? t + 1 : 0;
        for (int i = start; i < col_size; ++i) {
          if (iou_above(me, sme, cbox[i], carea[i], thresh)) bits |= 1ULL << i;
        }
        mask[((size_t)img * max_n + row) * col_blocks + cb] = bits;
      }
    }
  }
}

// One CTA per image walks the 64-box blocks in score order.  Thread 0 resolves the in-block
// chain from the diagonal words; all threads then OR the kept rows into the running
// suppression vector of the later blocks.  Stops as soon as max_keep boxes are kept.
__global__ void __launch_bounds__(256)
nms_scan_kernel(const u64 *__restrict__ mask, const int *__restrict__ counts, int max_n,
                int col_blocks, int max_keep, int keep_stride, int *__restrict__ keep_out,
                int *__restrict__ num_out, const int *__restrict__ gate) {
  extern __shared__ u64 remv[];
  if (gate && gate[blockIdx.x] == 0) return;
  __shared__ u64 diag[kNmsTile];
  __shared__ u64 s_kept;
  __shared__ int s_nkeep;
  __shared__ int s_rows[kNmsTile];     // in-block indices of the boxes kept in the current block
  const int img = blockIdx.x, tid = threadIdx.x;
  const int n = counts ? min(counts[img], max_n) : max_n;
  const int cb = (n + kNmsTile - 1) / kNmsTile;
  const u64 *m = mask + (size_t)img * max_n * col_blocks;
  int *keep = keep_out + (size_t)img * keep_stride;
  for (int j = tid; j < cb; j += blockDim.x) remv[j] = 0;
  if (tid == 0) s_nkeep = 0;
  __syncthreads();
  for (int blk = 0; blk < cb; ++blk) {
    const int base = blk * kNmsTile;
    if (tid < kNmsTile) {
      int r = base + tid;
      diag[tid] = (r < n) ? m[(size_t)r * col_blocks + blk] : 0ULL;
    }
    __syncthreads();
    if (tid == 0) {
      u64 cur = remv[blk], kept = 0;
      int nk = s_nkeep;
      const int lim = min(kNmsTile, n - base);
      for (int t = 0; t < lim; ++t) {
        if (!((cur >> t) & 1ULL)) {
          s_rows[__popcll(kept)] = t;
          kept |= 1ULL << t;
          if (nk < keep_stride) keep[nk] = base + t;
          ++nk;
          cur |= diag[t];
          if (max_keep > 0 && nk >= max_keep) break;
        }
      }
      s_kept = kept;
      s_nkeep = nk;
    }
    __syncthreads();
    const u64 kept = s_kept;
    if (max_keep > 0 && s_nkeep >= max_keep) break;
    if (kept) {
      // OR the mask rows of this block's kept boxes into the suppression words of the later blocks.  The row list is
      // walked eight at a time with the loads issued before any is consumed: one dependent load per kept box (the
      // earlier form) exposed a full L2 latency per box, ~0.3 us x 10 000 kept boxes.
      const int cnt = __popcll(kept);
      for (int j = blk + 1 + tid; j < cb; j += blockDim.x) {
        u64 acc = remv[j];
        const u64 *col = m + (size_t)base * col_blocks + j;
        for (int i = 0; i < cnt; i += 8) {
          u64 v[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) v[q] = (i + q < cnt) ? col[(size_t)s_rows[i + q] * col_blocks] : 0ULL;
#pragma unroll
          for (int q = 0; q < 8; ++q) acc |= v[q];
        }
        remv[j] = acc;
      }
    }
    __syncthreads();
  }
  if (tid == 0) num_out[img] = min(s_nkeep, keep_stride);
}

__global__ void extract_box4_kernel(const float *__restrict__ src, int n, int dim, float4 *__restrict__ dst) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float *p = src + (size_t)i * dim;
    dst[i] = make_float4(p[0], p[1], p[2], p[3]);
  }
}

static inline int nms_col_blocks(int max_n) { return (max_n + kNmsTile - 1) / kNmsTile; }

int nms_sorted_launch(const float *boxes, const int *counts, int batch, int max_n, float thresh,
                      int max_keep, int keep_stride, int *keep_out, int *num_out, void *workspace,
                      size_t workspace_bytes, cudaStream_t st, const int *gate) {
  if (batch <= 0 || max_n <= 0) return CTPN_OK;
  const int cb = nms_col_blocks(max_n);
  size_t need = (size_t)batch * max_n * cb * sizeof(u64);
  if (workspace_bytes < need) {
    set_error("ctpn_nms_sorted: workspace %zu < %zu bytes", workspace_bytes, need);
    return CTPN_ERR_WORKSPACE;
  }
  CTPN_REQUIRE(((uintptr_t)boxes & 15) == 0, "ctpn_nms_sorted: boxes must be 16-byte aligned");
  u64 *mask = reinterpret_cast<u64 *>(workspace);
  long long pairs = (long long)cb * cb;
  int sms = 0;
  if (int rc = current_sm_count(&sms)) return rc;
  const long long cap = 16ll * sms;        // grid-stride loop: 16 CTAs per SM
  const unsigned grid = (unsigned)(pairs < cap ? pairs : cap);
  ProfScope prof("nms (mask+scan)", 0.0, st);
  nms_mask_kernel<<<grid, kNmsTile, 0, st>>>(reinterpret_cast<const float4 *>(boxes), counts, batch, max_n, cb, thresh, mask, gate);
  CTPN_LAUNCH_CHECK();
  size_t smem = (size_t)cb * sizeof(u64);
  CTPN_REQUIRE(smem <= 200 * 1024, "ctpn_nms_sorted: %d boxes exceed the scan kernel's shared memory", max_n);
  if (smem > 48 * 1024)
    CTPN_CUDA(cudaFuncSetAttribute(nms_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  nms_scan_kernel<<<batch, 256, smem, st>>>(mask, counts, max_n, cb, max_keep, keep_stride, keep_out, num_out, gate);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

// ---- grow-only per-device scratch for the host entry point --------------------------------
struct HostNmsScratch {
  void *raw = nullptr, *box4 = nullptr, *mask = nullptr, *keep = nullptr;
  size_t raw_b = 0, box4_b = 0, mask_b = 0, keep_b = 0;
};
static HostNmsScratch g_scratch[64];
static std::mutex g_scratch_mu;

static int grow(void **p, size_t *cap, size_t need) {
  if (*cap >= need) return CTPN_OK;
  if (*p) CTPN_CUDA(cudaFree(*p));
  *p = nullptr;
  *cap = 0;
  size_t sz = align_up(need + need / 4, 256);
  CTPN_CUDA(cudaMalloc(p, sz));
  *cap = sz;
  return CTPN_OK;
}

}  // namespace ctpn

using namespace ctpn;

extern "C" size_t ctpn_nms_workspace_bytes(int batch, int max_n) {
  if (batch <= 0 || max_n <= 0) return 0;
  return (size_t)batch * max_n * nms_col_blocks(max_n) * sizeof(u64);
}

extern "C" int ctpn_nms_sorted(const float *boxes, const int *counts, int batch, int max_n, float thresh,
                               int max_keep, int *keep_out, int *num_out, void *workspace,
                               size_t workspace_bytes, void *stream) {
  CTPN_REQUIRE(boxes && keep_out && num_out, "ctpn_nms_sorted: null pointer");
  CTPN_REQUIRE(batch >= 0 && max_n >= 0, "ctpn_nms_sorted: negative size");
  int stride = max_keep > 0 ? max_keep : max_n;
  return nms_sorted_launch(boxes, counts, batch, max_n, thresh, max_keep, stride, keep_out, num_out, workspace,
                           workspace_bytes, (cudaStream_t)stream, nullptr);
}

extern "C" int ctpn_nms_host(int *keep_out, int *num_out, const float *boxes_host, int boxes_num, int boxes_dim,
                             float nms_overlap_thresh, int device_id) {
  CTPN_REQUIRE(keep_out && num_out, "ctpn_nms_host: null output pointer");
  CTPN_REQUIRE(boxes_num >= 0, "ctpn_nms_host: boxes_num < 0");
  *num_out = 0;
  if (boxes_num == 0) return CTPN_OK;
  CTPN_REQUIRE(boxes_host, "ctpn_nms_host: null boxes");
  CTPN_REQUIRE(boxes_dim >= 4, "ctpn_nms_host: boxes_dim must be >= 4 (got %d)", boxes_dim);
  CTPN_REQUIRE(device_id >= 0 && device_id < 64, "ctpn_nms_host: bad device id %d", device_id);
  int cur = -1;
  CTPN_CUDA(cudaGetDevice(&cur));
  if (cur != device_id) CTPN_CUDA(cudaSetDevice(device_id));   // nms_kernel.cu:80-89 semantics
  std::lock_guard<std::mutex> lock(g_scratch_mu);
  HostNmsScratch &s = g_scratch[device_id];
  const size_t n = boxes_num;
  int rc;
  if ((rc = grow(&s.raw, &s.raw_b, n * boxes_dim * sizeof(float)))) return rc;
  if ((rc = grow(&s.box4, &s.box4_b, n * sizeof(float4)))) return rc;
  if ((rc = grow(&s.mask, &s.mask_b, ctpn_nms_workspace_bytes(1, boxes_num)))) return rc;
  if ((rc = grow(&s.keep, &s.keep_b, (n + 1) * sizeof(int)))) return rc;
  cudaStream_t st = 0;
  CTPN_CUDA(cudaMemcpyAsync(s.raw, boxes_host, n * boxes_dim * sizeof(float), cudaMemcpyHostToDevice, st));
  extract_box4_kernel<<<ceil_div(boxes_num, 256), 256, 0, st>>>((const float *)s.raw, boxes_num, boxes_dim, (float4 *)s.box4);
  CTPN_LAUNCH_CHECK();
  int *keep_d = (int *)s.keep;
  int *num_d = keep_d + n;
  rc = nms_sorted_launch((const float *)s.box4, nullptr, 1, boxes_num, nms_overlap_thresh, 0, boxes_num, keep_d, num_d,
                         s.mask, s.mask_b, st, nullptr);
  if (rc) return rc;
  int num = 0;
  CTPN_CUDA(cudaMemcpyAsync(&num, num_d, sizeof(int), cudaMemcpyDeviceToHost, st));
  CTPN_CUDA(cudaStreamSynchronize(st));
  if (num > 0) CTPN_CUDA(cudaMemcpy(keep_out, keep_d, (size_t)num * sizeof(int), cudaMemcpyDeviceToHost));
  *num_out = num;
  return CTPN_OK;
}
