// Shared helpers for the ctpn_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/ctpn_b200.h"

namespace ctpn {

// ---- error plumbing ---------------------------------------------------------------------
void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what, const char *file, int line);
// SM count of the current device (cached per device): grid sizes follow the GPU the library runs on
int current_sm_count(int *sms);

#define CTPN_CUDA(call)                                                        \
  do {                                                                         \
    cudaError_t _e = (call);                                                   \
    if (_e != cudaSuccess) return ::ctpn::cuda_fail(_e, #call, __FILE__, __LINE__); \
  } while (0)

#define CTPN_REQUIRE(cond, ...)                \
  do {                                         \
    if (!(cond)) {                             \
      ::ctpn::set_error(__VA_ARGS__);          \
      return CTPN_ERR_INVALID;                 \
    }                                          \
  } while (0)

#define CTPN_LAUNCH_CHECK()                                                    \
  do {                                                                         \
    cudaError_t _e = cudaGetLastError();                                       \
    if (_e != cudaSuccess) return ::ctpn::cuda_fail(_e, "kernel launch", __FILE__, __LINE__); \
  } while (0)

// Optional per-launch timing: when enabled through ctpn_prof_enable(1), every instrumented launch is
// bracketed by CUDA events on its own stream; `work` is the algorithmic FLOPs (or bytes) of the launch.
bool prof_enabled();
struct ProfScope {
  ProfScope(const char *label, double work, cudaStream_t st);
  ~ProfScope();
  cudaStream_t st_;
  int idx_;
};

// ---- ragged batches (ctpn_net_forward_ragged) -----------------------------------------------
// The network stages with per-image extents: sizes = device int32 [B][2] full-resolution image sizes (h, w) of a batch
// whose canvas is [B][H][W]; a stage whose output is k pools down (shift = k) treats (h >> k, w >> k), clamped to its
// frame, as the image and stores zeros outside it.  sizes = nullptr is the uniform batch (the public entry points).
int conv1_1_tc_ragged(const void *src, int src_is_f32, const float *lut, const float *w_hwio, const float *bias, void *out_planes,
                      int B, int H, int W, int planes, bool outq, float out_s, float out_t, const int *sizes, void *stream);
// ctpn_conv3x3 (q = null) and ctpn_conv3x3_f16f8 (q = its scales, planes = 2) with the extents above (ext = sizes, ext_shift = shift)
struct QuantScales { float inv_main, inv_cross, out_s, out_t; };
int conv_tc_run(const void *in_planes, const void *w_planes, const float *bias, void *out, int B, int H, int W, int cin,
                int cout, int taps, int planes, int flags, const QuantScales *q, const int *ext, int ext_shift, void *stream);
// R = B * rows_per_image rows; row b * rows_per_image + y runs (h_b >> 4, w_b >> 4) steps and is zero outside them
int bilstm_ragged(const float *xproj, const float *wh_fw, const float *wh_bw, void *out_planes, int R, int W, int planes,
                  const int *sizes, int rows_per_image, void *stream);

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// ---- bf16 plane split -------------------------------------------------------------------
// a = p0 + p1 + p2 with p0 = bf16_rn(a), p1 = bf16_rn(a - p0), p2 = bf16_rn(a - p0 - p1).
__device__ __forceinline__ void split_planes(float a, int planes, __nv_bfloat16 *p) {
  __nv_bfloat16 h0 = __float2bfloat16_rn(a);
  p[0] = h0;
  if (planes > 1) {
    float r1 = __fsub_rn(a, __bfloat162float(h0));
    __nv_bfloat16 h1 = __float2bfloat16_rn(r1);
    p[1] = h1;
    if (planes > 2) {
      float r2 = __fsub_rn(r1, __bfloat162float(h1));
      p[2] = __float2bfloat16_rn(r2);
    }
  }
}

// Two floats -> P packed bf16 plane words (low half = plane of a, high half = plane of b).  One cvt.rn.bf16x2.f32 per
// plane; the exact residual for the next plane is formed from the halves of the packed word.  Same values as
// split_planes() on a and b separately.
template <int P>
__device__ __forceinline__ void split_planes2(float a, float b, uint32_t (&w)[P]) {
#pragma unroll
  for (int pl = 0; pl < P; ++pl) {
    uint32_t pk;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(pk) : "f"(b), "f"(a));   // first source -> upper half
    w[pl] = pk;
    if (pl + 1 < P) {
      a = __fsub_rn(a, __uint_as_float(pk << 16));
      b = __fsub_rn(b, __uint_as_float(pk & 0xffff0000u));
    }
  }
}

// ---- "F16F8" operand format (2 tensor-core units per MAC instead of the 3 of two bf16 planes) -----------------------
// A float32 value a is carried as  h = fp16_rn(a * s)  (11 significant bits) and its exact residual  r = a * s - h
// (|r| <= 2^-11 |h|).  A product a * w = (h_a + r_a)(h_w + r_w) / (s_a s_w) is evaluated as
//     main  = h_a * h_w                          fp16 wgmma (fp16 x fp16, exact products, fp32 accumulate): 1 unit
//     cross = q(h_a) * q(r_w) + q(r_a) * q(h_w)   e4m3 wgmma on e4m3 copies, K-concatenated: 2 x 1/2 unit
// (r_a * r_w ~ 2^-22 is dropped).  Storage per element: 2 B (h) + 1 B (e4m3 of a) + 1 B (e4m3 of r) = the 4 B of two bf16
// planes.  The e4m3 copies use per-tensor power-of-two scales t (values) and 2^11 t (residuals) so that both cross
// products carry the same scale: e4m3(a t_a) * e4m3(r_w 2^11 t_w) and e4m3(r_a 2^11 t_a) * e4m3(w t_w).
// Plane 0: fp16 [B][H][W][C].  Plane 1, per pixel and 64-channel block, 128 bytes: e4m3(a t)[64] | e4m3(r 2^11 t / s)[64]
// -- one 128-byte swizzle row = K 128 of the fp8 MMA (4 instructions of K = 32).
constexpr float kResidualGain = 2048.0f;      // 2^11

// (a, b) -> fp16x2 word (a in the low half), saturating; ra/rb receive the exact residuals a - h_a, b - h_b
__device__ __forceinline__ uint32_t f16x2_split(float a, float b, float &ra, float &rb) {
  uint32_t pk;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(pk) : "f"(b), "f"(a));   // first source -> upper half
  const __half2 h = *reinterpret_cast<const __half2 *>(&pk);
  ra = __fsub_rn(a, __low2float(h));
  rb = __fsub_rn(b, __high2float(h));
  return pk;
}
// four floats -> four e4m3 bytes (a in the lowest byte), saturating to +-448
__device__ __forceinline__ uint32_t e4m3x4(float a, float b, float c, float d) {
  uint16_t lo, hi;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
  return (uint32_t)lo | ((uint32_t)hi << 16);
}

// two round-to-nearest float32 products / fused multiply-adds on a pair of values
__device__ __forceinline__ float2 fmul2_rn(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 ffma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// four values -> their F16F8 words: two fp16x2 words (of v * s), e4m3x4 of v * t, e4m3x4 of the residuals * rs.
// s == 1 (no fp16 pre-scale, the usual case) skips its multiply.
__device__ __forceinline__ void f16f8_quad(float v0, float v1, float v2, float v3, float s, float t, float rs, uint32_t &h01,
                                           uint32_t &h23, uint32_t &qv, uint32_t &qr) {
  const float2 a = make_float2(v0, v1), b = make_float2(v2, v3);
  float2 as = a, bs = b;
  if (s != 1.f) {
    as = fmul2_rn(a, make_float2(s, s));
    bs = fmul2_rn(b, make_float2(s, s));
  }
  float2 ra, rb;
  h01 = f16x2_split(as.x, as.y, ra.x, ra.y);
  h23 = f16x2_split(bs.x, bs.y, rb.x, rb.y);
  const float2 at = fmul2_rn(a, make_float2(t, t)), bt = fmul2_rn(b, make_float2(t, t));
  qv = e4m3x4(at.x, at.y, bt.x, bt.y);
  ra = fmul2_rn(ra, make_float2(rs, rs));
  rb = fmul2_rn(rb, make_float2(rs, rs));
  qr = e4m3x4(ra.x, ra.y, rb.x, rb.y);
}

__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 lo, __nv_bfloat16 hi) {
  return (uint32_t)__bfloat16_as_ushort(lo) | ((uint32_t)__bfloat16_as_ushort(hi) << 16);
}

__device__ __forceinline__ float bf16_bits_to_float(uint32_t bits16) {
  return __uint_as_float(bits16 << 16);
}

}  // namespace ctpn
