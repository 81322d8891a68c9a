// BiLSTM recurrence over the feature-map width (lib/networks/network.py:93-101: LSTMCell(128)
// forward and backward over W for every feature-map row, zero initial state).
//
// The input projection x.Wx + b for both directions is a plain GEMM (done by ctpn_conv3x3 with
// taps = 1); this kernel runs the sequential part.  The recurrent matrix Wh is 128 x 512 float32
// = 256 KiB, more than one SM's shared memory, so a 2-CTA thread-block cluster splits the hidden
// units: CTA r keeps the 4 x 64 gate columns of units [64r, 64r+64) (128 KiB) resident in shared
// memory for the whole sequence and the two CTAs exchange their halves of h_t through
// distributed shared memory once per step.  Each cluster advances RG independent rows of one
// direction, so Wh is read from shared memory once per RG rows.  All arithmetic is float32; the mat-vec keeps even-k and
// odd-k partial sums (added at the end) so that one 16-byte weight load feeds two k.
//
// Ragged batches (sizes != null): row b * FH + y is a row of image b with (h_b >> 4, w_b >> 4) feature cells; it runs
// w_b >> 4 steps when y < h_b >> 4 (none otherwise), the backward direction starting at its own last column, and its outputs
// past that length are zero.  A cluster runs to the longest of its rows; each row's arithmetic is that of a uniform batch.
//
// TF 1.3 LSTMCell: gates (i, j, f, o) = [x, h] . kernel + bias;
//   c = sigmoid(f + 1) * c + sigmoid(i) * tanh(j);  h = sigmoid(o) * tanh(c).
#include <cooperative_groups.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace ctpn {

constexpr int kHid = 128, kGates = 512;

__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.0f / (1.0f + expf(-x)); }
// Cell non-linearities on the special-function unit (ex2.approx + rcp.approx, ~3e-7 absolute error) for the modes whose
// tolerance is >= 1e-5; the float32-equivalent mode (planes = 3) keeps expf / tanhf / IEEE division.  The accurate versions
// cost about as many instructions per step as the whole mat-vec.
template <bool FAST> __device__ __forceinline__ float lstm_sigmoid(float x) {
  return FAST ? __fdividef(1.0f, 1.0f + __expf(-x)) : sigmoidf_acc(x);
}
template <bool FAST> __device__ __forceinline__ float lstm_tanh(float x) {
  return FAST ? __fmaf_rn(2.0f, __fdividef(1.0f, 1.0f + __expf(-2.0f * x)), -1.0f) : tanhf(x);
}

// NC = CTAs per cluster: CTA `rank` owns hidden units [rank * 128/NC, (rank + 1) * 128/NC) and the 4 gate columns of each.
// NC = 2 is the product configuration; NC = 4 (64 KiB weight slice, two CTAs per SM) is a measured dead end kept for the
// test library only (see ctpn_bilstm_recurrent).
template <int RG, int NC, bool FAST>
__global__ void __launch_bounds__(256, NC == 4 ? 2 : 1)
bilstm_kernel(const float *__restrict__ xproj, const float *__restrict__ wh_fw, const float *__restrict__ wh_bw,
              __nv_bfloat16 *__restrict__ out, int R, int W, int planes, const int *__restrict__ sizes, int FH) {
  constexpr int kUnits = kHid / NC;          // hidden units of this CTA
  constexpr int kLocalCols = 4 * kUnits;     // their i, j, f, o gate columns
  constexpr int kCG = kLocalCols / 4;        // column groups (4 adjacent columns per thread)
  constexpr int kRGroups = 256 / kCG;        // row groups
  extern __shared__ __align__(16) float smem[];
  float *Ws = smem;                          // [128][kLocalCols]  recurrent weights of this CTA's units
  float *hbuf = Ws + kHid * kLocalCols;      // [2][RG][128] full hidden state, double buffered
  float *gates = hbuf + 2 * RG * kHid;       // [RG][256]    pre-activations of this CTA's columns
  __shared__ int len[RG];                    // sequence length of each row of the group (0: no row / a dead row)
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  static_assert(NC == 2 || NC == 4, "cluster of 2 or 4 CTAs");
  const int cid = blockIdx.x / NC;                       // cluster index
  const int groups = (R + RG - 1) / RG;
  const int dir = cid / groups, row0 = (cid % groups) * RG;
  const int t = threadIdx.x;
  // mat-vec phase: thread = 4 adjacent local columns x RG/4 rows (register tile: 4 + RG/4 shared-memory loads
  // per 4 * RG/4 * 4 FMAs); cell phase: thread = unit ul, rows (t >> 6) + 4q
  constexpr int RT = RG / kRGroups;
  static_assert(RT >= 1 && RT * kRGroups == RG, "RG must be a multiple of the row-group count");
  const int cg = t % kCG, rg = t / kCG;                  // column group (4 columns), row group (RT rows)
  const int lc0 = cg * 4;                                // first local column; gate = lc0 / kUnits, unit = lc0 % kUnits
  const int gcol0 = (lc0 / kUnits) * kHid + rank * kUnits + (lc0 % kUnits);   // column in the 512-wide gate vector
  const int ul = t % kUnits;
  const float *wh = dir ? wh_bw : wh_fw;
  // Shared-memory layout of the weights for the paired FMAs: [column pair half][k pair][column group][4] with
  // the 4 floats = (col a: k even, k odd; col b: k even, k odd), so one LDS.128 hands a thread two (k, k+1) weight
  // pairs and consecutive lanes read consecutive 16-byte chunks (conflict-free).
  for (int i = t; i < kHid * kLocalCols; i += 256) {
    const int k = i / kLocalCols, lc = i % kLocalCols;
    const int cgi = lc >> 2, cc = lc & 3;
    Ws[(((cc >> 1) * (kHid / 2) + (k >> 1)) * kCG + cgi) * 4 + (cc & 1) * 2 + (k & 1)] =
        wh[k * kGates + (lc / kUnits) * kHid + rank * kUnits + (lc % kUnits)];
  }
  for (int i = t; i < 2 * RG * kHid; i += 256) hbuf[i] = 0.f;
  if (t < RG) {
    const int row = row0 + t;
    int n = row < R ? W : 0;
    if (sizes && row < R) {      // clamped to the canvas: a wrong size never addresses outside it
      const int b = row / FH, y = row - b * FH;
      n = y < min(FH, __ldg(sizes + 2 * b) >> 4) ? max(0, min(W, __ldg(sizes + 2 * b + 1) >> 4)) : 0;
    }
    len[t] = n;
  }
  float *peer_h[NC];
#pragma unroll
  for (int r = 0; r < NC; ++r) peer_h[r] = cluster.map_shared_rank(hbuf, r);
  constexpr int kCellRows = RG / (256 / kUnits);         // rows per thread in the cell phase
  float c_state[kCellRows];
#pragma unroll
  for (int q = 0; q < kCellRows; ++q) c_state[q] = 0.f;
  cluster.sync();
  int steps = 0;
  for (int r = 0; r < RG; ++r) steps = max(steps, len[r]);

  const long long plane_stride = (long long)R * W * 2 * kHid;
  float4 xnext[RT];
#pragma unroll
  for (int r = 0; r < RT; ++r) {
    const int row = row0 + rg * RT + r, n = len[rg * RT + r];
    xnext[r] = n > 0 ? __ldg(reinterpret_cast<const float4 *>(xproj + ((long long)row * W + (dir ? n - 1 : 0)) * (2 * kGates) + dir * kGates + gcol0))
                     : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int step = 0; step < steps; ++step) {
    const float *hc = hbuf + (step & 1) * RG * kHid;
    const int hn_off = ((step + 1) & 1) * RG * kHid;
    // acc[r][c] = (sum over even k, sum over odd k) for local column lc0 + c: each ffma2_rn advances two k at once with the
    // natural register pairs (h[k], h[k+1]) x (w[k][c], w[k+1][c]).
    float2 acc[RT][4];
#pragma unroll
    for (int r = 0; r < RT; ++r) {
      const float4 x = xnext[r];
      acc[r][0] = make_float2(x.x, 0.f); acc[r][1] = make_float2(x.y, 0.f);
      acc[r][2] = make_float2(x.z, 0.f); acc[r][3] = make_float2(x.w, 0.f);
    }
    if (step + 1 < steps) {   // x-projection of the next step: in flight during this step's mat-vec
#pragma unroll
      for (int r = 0; r < RT; ++r) {
        const int row = row0 + rg * RT + r, n = len[rg * RT + r];
        const int tn = dir ? n - 2 - step : step + 1;
        if (step + 1 < n) xnext[r] = __ldg(reinterpret_cast<const float4 *>(xproj + ((long long)row * W + tn) * (2 * kGates) + dir * kGates + gcol0));
      }
    }
    const float4 *w_lo = reinterpret_cast<const float4 *>(Ws) + cg;                       // columns lc0, lc0 + 1
    const float4 *w_hi = reinterpret_cast<const float4 *>(Ws) + (kHid / 2) * kCG + cg;    // columns lc0 + 2, lc0 + 3
#pragma unroll 2
    for (int k = 0; k < kHid; k += 4) {
      const float4 wa0 = w_lo[(k >> 1) * kCG], wa1 = w_lo[((k >> 1) + 1) * kCG];
      const float4 wb0 = w_hi[(k >> 1) * kCG], wb1 = w_hi[((k >> 1) + 1) * kCG];
#pragma unroll
      for (int r = 0; r < RT; ++r) {
        const float4 h4 = *reinterpret_cast<const float4 *>(hc + (rg * RT + r) * kHid + k);
        const float2 h01 = make_float2(h4.x, h4.y), h23 = make_float2(h4.z, h4.w);
        acc[r][0] = ffma2_rn(h01, make_float2(wa0.x, wa0.y), acc[r][0]);
        acc[r][1] = ffma2_rn(h01, make_float2(wa0.z, wa0.w), acc[r][1]);
        acc[r][2] = ffma2_rn(h01, make_float2(wb0.x, wb0.y), acc[r][2]);
        acc[r][3] = ffma2_rn(h01, make_float2(wb0.z, wb0.w), acc[r][3]);
        acc[r][0] = ffma2_rn(h23, make_float2(wa1.x, wa1.y), acc[r][0]);
        acc[r][1] = ffma2_rn(h23, make_float2(wa1.z, wa1.w), acc[r][1]);
        acc[r][2] = ffma2_rn(h23, make_float2(wb1.x, wb1.y), acc[r][2]);
        acc[r][3] = ffma2_rn(h23, make_float2(wb1.z, wb1.w), acc[r][3]);
      }
    }
#pragma unroll
    for (int r = 0; r < RT; ++r)
      *reinterpret_cast<float4 *>(gates + (rg * RT + r) * kLocalCols + lc0) =
          make_float4(acc[r][0].x + acc[r][0].y, acc[r][1].x + acc[r][1].y, acc[r][2].x + acc[r][2].y, acc[r][3].x + acc[r][3].y);
    __syncthreads();
    // cell update: thread -> unit ul, rows (t / kUnits) + (256 / kUnits) * q
#pragma unroll
    for (int q = 0; q < kCellRows; ++q) {
      const int r = (t / kUnits) + (256 / kUnits) * q;
      const float gi = gates[r * kLocalCols + ul], gj = gates[r * kLocalCols + kUnits + ul];
      const float gf = gates[r * kLocalCols + 2 * kUnits + ul], go = gates[r * kLocalCols + 3 * kUnits + ul];
      const float c = lstm_sigmoid<FAST>(gf + 1.0f) * c_state[q] + lstm_sigmoid<FAST>(gi) * lstm_tanh<FAST>(gj);
      const float h = lstm_sigmoid<FAST>(go) * lstm_tanh<FAST>(c);
      c_state[q] = c;
      const int u = rank * kUnits + ul;
#pragma unroll
      for (int pr = 0; pr < NC; ++pr) peer_h[pr][hn_off + r * kHid + u] = h;     // own copy and every peer's (DSMEM)
      const int row = row0 + r, n = len[r];
      if (row < R) {     // a row past its length writes a zero at column `step` instead (columns >= steps: below)
        __nv_bfloat16 pl[3];
        split_planes(step < n ? h : 0.f, planes, pl);
        const int tpos = step >= n ? step : dir ? n - 1 - step : step;
        const long long o = ((long long)row * W + tpos) * (2 * kHid) + dir * kHid + u;
        for (int p = 0; p < planes; ++p) out[p * plane_stride + o] = pl[p];
      }
    }
    cluster.sync();   // h_{t} of both halves visible in both CTAs; also orders the gates[] reuse
  }
  // ragged batch: the columns past the group's longest row are zero
  for (int step = steps; step < W; ++step) {
#pragma unroll
    for (int q = 0; q < kCellRows; ++q) {
      const int row = row0 + (t / kUnits) + (256 / kUnits) * q;
      if (row < R) {
        const long long o = ((long long)row * W + step) * (2 * kHid) + dir * kHid + rank * kUnits + ul;
        for (int p = 0; p < planes; ++p) out[p * plane_stride + o] = __float2bfloat16_rn(0.f);
      }
    }
  }
}

template <int RG, int NC>
static int launch_bilstm(const float *xproj, const float *wh_fw, const float *wh_bw, void *out, int R, int W, int planes,
                         const int *sizes, int FH, cudaStream_t st) {
  constexpr int kLocalCols = 4 * kHid / NC;
  const size_t smem = (size_t)(kHid * kLocalCols + 2 * RG * kHid + RG * kLocalCols) * sizeof(float);
  auto kernel = planes <= 2 ? bilstm_kernel<RG, NC, true> : bilstm_kernel<RG, NC, false>;
  CTPN_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int groups = (R + RG - 1) / RG;
  ProfScope prof("bilstm_recurrent", 2.0 * 2.0 * R * W * 128.0 * 512.0, st);
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = NC; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
  cfg.gridDim = dim3(NC * 2 * groups);
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  CTPN_CUDA(cudaLaunchKernelEx(&cfg, kernel, xproj, wh_fw, wh_bw, (__nv_bfloat16 *)out, R, W, planes, sizes, FH));
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

}  // namespace ctpn

using namespace ctpn;

extern "C" int ctpn_bilstm_recurrent(const float *xproj, const float *wh_fw, const float *wh_bw, void *out_planes, int R,
                                     int W, int planes, void *stream) {
  return bilstm_ragged(xproj, wh_fw, wh_bw, out_planes, R, W, planes, nullptr, R, stream);
}

int ctpn::bilstm_ragged(const float *xproj, const float *wh_fw, const float *wh_bw, void *out_planes, int R, int W, int planes,
                        const int *sizes, int FH, void *stream) {
  CTPN_REQUIRE(xproj && wh_fw && wh_bw && out_planes, "ctpn_bilstm_recurrent: null pointer");
  CTPN_REQUIRE(R > 0 && W > 0 && FH > 0, "ctpn_bilstm_recurrent: bad shape R=%d W=%d", R, W);
  CTPN_REQUIRE(planes >= 1 && planes <= 3, "ctpn_bilstm_recurrent: planes must be 1..3");
  cudaStream_t st = (cudaStream_t)stream;
  // Rows per cluster (RG): the fewest that still run every cluster in ONE wave.  A CTA holds 130-210 KiB of shared memory,
  // so one CTA per SM and SMs / 4 clusters per direction in a wave; a second wave would repeat all W steps, while fewer
  // rows per cluster shorten each step.  RG = 40 (208 KiB) is the largest slice that fits; beyond 40 x SMs / 4 rows the
  // launch takes more than one wave.  On 132 SMs, batch 32 x 600x900 (R = 1184) runs at RG = 40: 30 clusters per direction.
  // The 4-CTA-cluster variant (two CTAs per SM, 16 warps) re-reads the weight slice once per row group, so two CTAs per SM
  // double the shared-memory traffic, and the h exchange and the cluster barrier span four CTAs; it stays selectable in
  // the test library (CTPN_LSTM_NC=4) for comparison.
  int sms = 0;
  if (int rc = current_sm_count(&sms)) return rc;
  const int per_wave = sms / 4 > 1 ? sms / 4 : 1;                  // 2-CTA clusters of each direction in one wave
  auto fits = [&](int rg) { return (R + rg - 1) / rg <= per_wave; };
#ifdef CTPN_DEBUG
  static const int force_nc = [] { const char *e = getenv("CTPN_LSTM_NC"); return e ? atoi(e) : 0; }();
  if (!fits(16) && force_nc == 4) return launch_bilstm<32, 4>(xproj, wh_fw, wh_bw, out_planes, R, W, planes, sizes, FH, st);
#endif
  if (fits(4)) return launch_bilstm<4, 2>(xproj, wh_fw, wh_bw, out_planes, R, W, planes, sizes, FH, st);
  if (fits(8)) return launch_bilstm<8, 2>(xproj, wh_fw, wh_bw, out_planes, R, W, planes, sizes, FH, st);
  if (fits(16)) return launch_bilstm<16, 2>(xproj, wh_fw, wh_bw, out_planes, R, W, planes, sizes, FH, st);
  if (fits(32)) return launch_bilstm<32, 2>(xproj, wh_fw, wh_bw, out_planes, R, W, planes, sizes, FH, st);
  return launch_bilstm<40, 2>(xproj, wh_fw, wh_bw, out_planes, R, W, planes, sizes, FH, st);
}
