// float32 SIMT reference kernels (test library only: libctpn_b200_dbg.so; not in the product library):
//   * ctpn_conv1_1        first VGG layer (Cin = 3, K = 27: HBM-bound, no tensor cores); fuses the
//                         uint8 -> float32 mean subtraction of lib/fast_rcnn/test.py:8-9
//   * ctpn_conv3x3_simt   same contract as ctpn_conv3x3 with plain float32 FMAs: the in-library
//                         reference the tests use to validate the wgmma kernel
// Reference semantics: lib/networks/network.py:160-196.
#include "../common.cuh"
#include "ctpn_b200_testing.h"

namespace ctpn {

// ---- conv1_1 ----------------------------------------------------------------------------------
// Lane = one pair of output channels (its 27 x 2 weights live in registers), warp = one tile row, and each
// pass computes 4 horizontally adjacent pixels from 3 x 18 input floats fetched with broadcast LDS.128:
// 216 FMAs per 15 shared-memory loads.  A warp's store covers one pixel x 64 channels = 128 contiguous
// bytes per plane.  The layer is HBM-write bound: 64 channels x P planes x 2 B per pixel out for 3 B in.
constexpr int kC1TileW = 32, kC1TileH = 8, kC1Threads = 256, kC1Row = 104;   // row pitch: 34 * 3 floats padded to 16 B

template <bool SRC_F32>
__global__ void __launch_bounds__(kC1Threads, 2)
conv1_1_kernel(const void *__restrict__ src, const float *__restrict__ lut, const float *__restrict__ w,
               const float *__restrict__ bias, __nv_bfloat16 *__restrict__ out, int B, int H, int W, int planes) {
  __shared__ __align__(16) float s_in[kC1TileH + 2][kC1Row];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.z;
  const int x0 = blockIdx.x * kC1TileW, y0 = blockIdx.y * kC1TileH;
  float wr[27][2];
#pragma unroll
  for (int k = 0; k < 27; ++k) {
    const float2 v = __ldg(reinterpret_cast<const float2 *>(w + k * 64 + lane * 2));
    wr[k][0] = v.x; wr[k][1] = v.y;
  }
  const float2 bv = __ldg(reinterpret_cast<const float2 *>(bias + lane * 2));
  for (int i = tid; i < (kC1TileH + 2) * (kC1TileW + 2) * 3; i += kC1Threads) {
    const int xc = i % ((kC1TileW + 2) * 3), yy = i / ((kC1TileW + 2) * 3);
    const int c = xc % 3, xx = xc / 3;
    const int gx = x0 + xx - 1, gy = y0 + yy - 1;
    float v = 0.f;   // SAME padding pads the mean-subtracted blob with zeros
    if (gx >= 0 && gx < W && gy >= 0 && gy < H) {
      const size_t off = (((size_t)b * H + gy) * W + gx) * 3 + c;
      if (SRC_F32) v = reinterpret_cast<const float *>(src)[off];
      else v = lut[reinterpret_cast<const uint8_t *>(src)[off] * 3 + c];
    }
    s_in[yy][xc] = v;
  }
  __syncthreads();
  const size_t plane_stride = (size_t)B * H * W * 64;
  const int y = y0 + warp;
  if (y >= H) return;
#pragma unroll 1
  for (int g = 0; g < kC1TileW / 4; ++g) {
    float in[3][20];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const float4 *row = reinterpret_cast<const float4 *>(&s_in[warp + ky][12 * g]);
#pragma unroll
      for (int q = 0; q < 5; ++q) {       // 18 floats needed; the 5th vector over-reads 2 floats of padding / next pixels
        const float4 v = row[q];
        in[ky][4 * q] = v.x; in[ky][4 * q + 1] = v.y; in[ky][4 * q + 2] = v.z; in[ky][4 * q + 3] = v.w;
      }
    }
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      float a0 = 0.f, a1 = 0.f;
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx)
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const float v = in[ky][(px + kx) * 3 + c];
            const int k = (ky * 3 + kx) * 3 + c;
            a0 = fmaf(v, wr[k][0], a0);
            a1 = fmaf(v, wr[k][1], a1);
          }
      const int x = x0 + 4 * g + px;
      if (x < W) {
        a0 = fmaxf(a0 + bv.x, 0.f);
        a1 = fmaxf(a1 + bv.y, 0.f);
        const size_t o = (((size_t)b * H + y) * W + x) * 64 + lane * 2;
        for (int p = 0; p < planes; ++p) {
          const __nv_bfloat16 h0 = __float2bfloat16_rn(a0), h1 = __float2bfloat16_rn(a1);
          *reinterpret_cast<uint32_t *>(out + p * plane_stride + o) = pack_bf16x2(h0, h1);
          a0 = __fsub_rn(a0, __bfloat162float(h0));
          a1 = __fsub_rn(a1, __bfloat162float(h1));
        }
      }
    }
  }
}

// ---- generic float32 SIMT conv on planes --------------------------------------------------------
// Block: 64 output pixels x 64 output channels, 256 threads (4 x 4 micro-tile each), K in chunks
// of 32 channels of one tap.  With CTPN_F_POOL the 4 positions of each 2x2 window are evaluated
// one after the other and max-reduced (4x the loads; this kernel is a reference, not the product).
constexpr int kSM = 64, kSN = 64, kSK = 32;

__device__ __forceinline__ float load_planes(const __nv_bfloat16 *p, long long off, long long plane_stride, int planes) {
  float v = __bfloat162float(p[off]);
  if (planes > 1) v += __bfloat162float(p[off + plane_stride]);
  if (planes > 2) v += __bfloat162float(p[off + 2 * plane_stride]);
  return v;
}

__global__ void __launch_bounds__(256)
conv_simt_kernel(const __nv_bfloat16 *__restrict__ in, const __nv_bfloat16 *__restrict__ wt,
                 const float *__restrict__ bias, void *__restrict__ out, int B, int H, int W, int Cin, int Cout,
                 int taps, int planes, int flags) {
  __shared__ float As[kSK][kSM + 4];
  __shared__ float Bs[kSK][kSN + 4];
  const bool pool = flags & CTPN_F_POOL;
  const int Ho = pool ? H / 2 : H, Wo = pool ? W / 2 : W;
  const long long M = (long long)B * Ho * Wo;
  const long long m0 = (long long)blockIdx.x * kSM;
  const int n0 = blockIdx.y * kSN;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const long long in_plane = (long long)B * H * W * Cin;
  const long long w_plane = (long long)Cout * taps * Cin;
  float best[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) best[i][j] = -INFINITY;
  const int nsub = pool ? 4 : 1;
  for (int sub = 0; sub < nsub; ++sub) {
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int tap = 0; tap < taps; ++tap) {
      const int dy = taps == 9 ? tap / 3 - 1 : 0, dx = taps == 9 ? tap % 3 - 1 : 0;
      for (int c0 = 0; c0 < Cin; c0 += kSK) {
        for (int e = tid; e < kSM * kSK; e += 256) {
          const int k = e % kSK, pm = e / kSK;
          const long long mm = m0 + pm;
          float v = 0.f;
          if (mm < M) {
            const int ox = (int)(mm % Wo), oy = (int)((mm / Wo) % Ho), b = (int)(mm / ((long long)Wo * Ho));
            const int y = (pool ? 2 * oy + (sub >> 1) : oy) + dy, x = (pool ? 2 * ox + (sub & 1) : ox) + dx;
            if (y >= 0 && y < H && x >= 0 && x < W)
              v = load_planes(in, (((long long)b * H + y) * W + x) * Cin + c0 + k, in_plane, planes);
          }
          As[k][pm] = v;
        }
        for (int e = tid; e < kSN * kSK; e += 256) {
          const int k = e % kSK, pn = e / kSK;
          Bs[k][pn] = load_planes(wt, ((long long)(n0 + pn) * taps + tap) * Cin + c0 + k, w_plane, planes);
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < kSK; ++k) {
          const float4 a = *reinterpret_cast<const float4 *>(&As[k][ty * 4]);
          const float4 bb = *reinterpret_cast<const float4 *>(&Bs[k][tx * 4]);
          const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) best[i][j] = fmaxf(best[i][j], acc[i][j]);
  }
  const long long out_plane = M * Cout;
  for (int i = 0; i < 4; ++i) {
    const long long mm = m0 + ty * 4 + i;
    if (mm >= M) continue;
    for (int j = 0; j < 4; ++j) {
      const int co = n0 + tx * 4 + j;
      float v = best[i][j] + bias[co];
      if (flags & CTPN_F_RELU) v = fmaxf(v, 0.f);
      if (flags & CTPN_F_OUT_F32) {
        reinterpret_cast<float *>(out)[mm * Cout + co] = v;
      } else {
        __nv_bfloat16 pl[3];
        split_planes(v, planes, pl);
        for (int p = 0; p < planes; ++p) reinterpret_cast<__nv_bfloat16 *>(out)[p * out_plane + mm * Cout + co] = pl[p];
      }
    }
  }
}

}  // namespace ctpn

using namespace ctpn;

extern "C" int ctpn_conv1_1(const void *src, int src_is_f32, const float *lut, const float *w_hwio, const float *bias,
                            void *out_planes, int B, int H, int W, int planes, void *stream) {
  CTPN_REQUIRE(src && w_hwio && bias && out_planes, "ctpn_conv1_1: null pointer");
  CTPN_REQUIRE(src_is_f32 || lut, "ctpn_conv1_1: uint8 input needs the mean-subtraction LUT");
  CTPN_REQUIRE(B > 0 && B <= 65535 && H > 0 && W > 0, "ctpn_conv1_1: bad shape");
  CTPN_REQUIRE(planes >= 1 && planes <= 3, "ctpn_conv1_1: planes must be 1..3");
  dim3 grid(ceil_div(W, kC1TileW), ceil_div(H, kC1TileH), B), block(kC1Threads);
  ProfScope prof("conv1_1", 2.0 * B * H * W * 27.0 * 64.0, (cudaStream_t)stream);
  if (src_is_f32)
    conv1_1_kernel<true><<<grid, block, 0, (cudaStream_t)stream>>>(src, lut, w_hwio, bias, (__nv_bfloat16 *)out_planes, B, H, W, planes);
  else
    conv1_1_kernel<false><<<grid, block, 0, (cudaStream_t)stream>>>(src, lut, w_hwio, bias, (__nv_bfloat16 *)out_planes, B, H, W, planes);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

extern "C" int ctpn_conv3x3_simt(const void *in_planes, const void *w_planes, const float *bias, void *out, int B,
                                 int H, int W, int cin, int cout, int taps, int planes, int flags, void *stream) {
  CTPN_REQUIRE(in_planes && w_planes && bias && out, "ctpn_conv3x3_simt: null pointer");
  CTPN_REQUIRE(taps == 9 || taps == 1, "ctpn_conv3x3_simt: taps must be 9 or 1");
  CTPN_REQUIRE(planes >= 1 && planes <= 3, "ctpn_conv3x3_simt: planes must be 1..3");
  CTPN_REQUIRE(cin % kSK == 0 && cout % kSN == 0, "ctpn_conv3x3_simt: Cin %% 32 and Cout %% 64 must be 0");
  const bool pool = flags & CTPN_F_POOL;
  const long long M = (long long)B * (pool ? H / 2 : H) * (pool ? W / 2 : W);
  dim3 grid((unsigned)((M + kSM - 1) / kSM), cout / kSN);
  ProfScope prof("conv_simt", 2.0 * B * H * W * (double)taps * cin * cout, (cudaStream_t)stream);
  conv_simt_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)in_planes, (const __nv_bfloat16 *)w_planes,
                                                           bias, out, B, H, W, cin, cout, taps, planes, flags);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}
