// Image front-end: cv2.resize(..., INTER_LINEAR) for uint8 images on the device, bit-exact with OpenCV's fixed-point
// path -- the arithmetic of the reference's resize_im (ctpn/demo.py:21-25; opencv-python is an un-vendored dependency,
// algorithm restated and pinned against cv2 in oracle/resize.py + tests/test_resize_cpu.py):
//   taps   f = float((d + 0.5) * scale - 0.5), s = floor(f), f -= s; columns drop the fraction at the border, rows
//          clamp both taps to the border row instead; weights cvRound((1 - f) * 2048), cvRound(f * 2048)
//   value  (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2 with r = s0 * a0 + s1 * a1 (int32)
//   exact 1/2 scale in both directions: INTER_AREA (rounded 2x2 mean; partial border blocks: mean of what exists)
// HBM-bound: one thread per output pixel, taps recomputed in registers (no coefficient tables), 4 gathers per channel
// served by L1/L2.
//
// ctpn_image_blob_f32: the float32 rescale of _get_image_blob (lib/fast_rcnn/test.py:7-31: `im_orig -= PIXEL_MEANS`, then
// cv2.resize of the FLOAT32 image by im_scale) fused with the mean subtraction.  OpenCV's own float path (resize.cpp,
// HResizeLinear / VResizeLinear without intrinsics reordering; pinned in oracle/resize.py against cv2 with IPP disabled):
//   taps as above but kept as float weights (1 - f, f); rows = S[sx] * a0 + S[sx + 1] * a1 and out = R0 * b0 + R1 * b1,
//   every product and sum rounded to float32 (no FMA); exact 1/2 scale: (((s00 + s01) + s10) + s11) * 0.25f.
// opencv-python wheels dispatch float32 INTER_LINEAR to Intel IPP, whose closed arithmetic differs from OpenCV's own code
// by up to ~1.4e-2 on 8-bit-range data for a 1100-px-wide image (tests/test_resize_cpu.py measures it), so "equal to cv2.resize" is build-dependent
// for float images; this kernel is bit-exact with the open implementation.
#include "common.cuh"

namespace ctpn {

__device__ __forceinline__ void resize_taps(int d, int sn, double scale, bool drop_border_fraction, int &s0, int &s1,
                                            int &w0, int &w1) {
  float f = (float)__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5);
  int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  if (drop_border_fraction) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= sn - 1) { f = 0.f; s = sn - 1; }
  }
  w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  w1 = __float2int_rn(__fmul_rn(f, 2048.f));
  s0 = min(max(s, 0), sn - 1);
  s1 = min(max(s + 1, 0), sn - 1);
}

__global__ void __launch_bounds__(256)
resize_linear_u8_kernel(const uint8_t *__restrict__ src, uint8_t *__restrict__ dst, int B, int sh, int sw, int C, int dh,
                        int dw, double scale_x, double scale_y, int area2) {
  const long long total = (long long)B * dh * dw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int dx = (int)(i % dw), dy = (int)((i / dw) % dh), b = (int)(i / ((long long)dw * dh));
    const uint8_t *im = src + (size_t)b * sh * sw * C;
    uint8_t *o = dst + (size_t)i * C;
    if (area2) {
      const int y0 = 2 * dy, x0 = 2 * dx;
      const int ny = min(2, sh - y0), nx = min(2, sw - x0);
      for (int c = 0; c < C; ++c) {
        int sum = 0;
        for (int yy = 0; yy < ny; ++yy)
          for (int xx = 0; xx < nx; ++xx) sum += im[((size_t)(y0 + yy) * sw + x0 + xx) * C + c];
        int v = (ny * nx == 4) ? (sum + 2) >> 2 : __float2int_rn(__fdiv_rn((float)sum, (float)(ny * nx)));
        o[c] = (uint8_t)min(max(v, 0), 255);
      }
      continue;
    }
    int sx0, sx1, a0, a1, sy0, sy1, b0, b1;
    resize_taps(dx, sw, scale_x, true, sx0, sx1, a0, a1);
    resize_taps(dy, sh, scale_y, false, sy0, sy1, b0, b1);
    const uint8_t *r0 = im + (size_t)sy0 * sw * C, *r1 = im + (size_t)sy1 * sw * C;
    for (int c = 0; c < C; ++c) {
      const int h0 = r0[(size_t)sx0 * C + c] * a0 + r0[(size_t)sx1 * C + c] * a1;
      const int h1 = r1[(size_t)sx0 * C + c] * a0 + r1[(size_t)sx1 * C + c] * a1;
      const int v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
      o[c] = (uint8_t)min(max(v, 0), 255);
    }
  }
}

// source coordinate and fractional weight of destination index d (float path)
__device__ __forceinline__ void resize_taps_f32(int d, int sn, double scale, bool drop_border_fraction, int &s0, int &s1,
                                                float &w0, float &w1) {
  float f = (float)__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5);
  int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  if (drop_border_fraction) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= sn - 1) { f = 0.f; s = sn - 1; }
  }
  w0 = __fsub_rn(1.f, f);
  w1 = f;
  s0 = min(max(s, 0), sn - 1);
  s1 = min(max(s + 1, 0), sn - 1);
}

// uint8 BGR image -> mean-subtracted float32 blob at another scale (3 channels; lut[256][3] = float32(double(v) - mean[c]))
__global__ void __launch_bounds__(256)
image_blob_f32_kernel(const uint8_t *__restrict__ src, const float *__restrict__ lut, float *__restrict__ dst, int B, int sh,
                      int sw, int dh, int dw, double scale_x, double scale_y, int area2) {
  const long long total = (long long)B * dh * dw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int dx = (int)(i % dw), dy = (int)((i / dw) % dh), b = (int)(i / ((long long)dw * dh));
    const uint8_t *im = src + (size_t)b * sh * sw * 3;
    float *o = dst + (size_t)i * 3;
    auto px = [&](int y, int x, int c) { return __ldg(lut + im[((size_t)y * sw + x) * 3 + c] * 3 + c); };
    if (area2) {
      const int y0 = 2 * dy, x0 = 2 * dx;
      const int ny = min(2, sh - y0), nx = min(2, sw - x0);
      for (int c = 0; c < 3; ++c) {
        float sum = px(y0, x0, c);
        if (nx == 2) sum = __fadd_rn(sum, px(y0, x0 + 1, c));
        if (ny == 2) {
          sum = __fadd_rn(sum, px(y0 + 1, x0, c));
          if (nx == 2) sum = __fadd_rn(sum, px(y0 + 1, x0 + 1, c));
        }
        o[c] = ny * nx == 4 ? __fmul_rn(sum, 0.25f) : __fdiv_rn(sum, (float)(ny * nx));
      }
      continue;
    }
    int sx0, sx1, sy0, sy1;
    float a0, a1, b0, b1;
    resize_taps_f32(dx, sw, scale_x, true, sx0, sx1, a0, a1);
    resize_taps_f32(dy, sh, scale_y, false, sy0, sy1, b0, b1);
    for (int c = 0; c < 3; ++c) {
      const float r0 = __fadd_rn(__fmul_rn(px(sy0, sx0, c), a0), __fmul_rn(px(sy0, sx1, c), a1));
      const float r1 = __fadd_rn(__fmul_rn(px(sy1, sx0, c), a0), __fmul_rn(px(sy1, sx1, c), a1));
      o[c] = __fadd_rn(__fmul_rn(r0, b0), __fmul_rn(r1, b1));
    }
  }
}

static int cv_round_host(double v) { return (int)nearbyint(v); }   // default rounding mode: half to even, like cvRound

}  // namespace ctpn

using namespace ctpn;

extern "C" int ctpn_resize_out_size(int sh, int sw, double fx, double fy, int *dh, int *dw) {
  CTPN_REQUIRE(dh && dw && sh > 0 && sw > 0 && fx > 0 && fy > 0, "ctpn_resize_out_size: bad arguments");
  *dh = cv_round_host((double)sh * fy);
  *dw = cv_round_host((double)sw * fx);
  CTPN_REQUIRE(*dh > 0 && *dw > 0, "ctpn_resize_out_size: empty result (%d x %d)", *dh, *dw);
  return CTPN_OK;
}

extern "C" int ctpn_resize_linear_u8(const void *src, int B, int sh, int sw, int channels, double fx, double fy, void *dst,
                                     int dh, int dw, void *stream) {
  CTPN_REQUIRE(src && dst, "ctpn_resize_linear_u8: null pointer");
  CTPN_REQUIRE(B > 0 && sh > 0 && sw > 0 && channels > 0 && channels <= 4, "ctpn_resize_linear_u8: bad shape");
  int eh = 0, ew = 0;
  int rc = ctpn_resize_out_size(sh, sw, fx, fy, &eh, &ew);
  if (rc) return rc;
  CTPN_REQUIRE(eh == dh && ew == dw, "ctpn_resize_linear_u8: dst is %d x %d, cv2 would produce %d x %d", dh, dw, eh, ew);
  const double scale_x = 1.0 / fx, scale_y = 1.0 / fy;
  const int area2 = (scale_x == 2.0 && scale_y == 2.0) ? 1 : 0;   // cv::resize routes exact 2x decimation to INTER_AREA
  const long long total = (long long)B * dh * dw;
  int sms = 0;
  if ((rc = current_sm_count(&sms))) return rc;
  const int grid = (int)std::min<long long>((total + 255) / 256, 32LL * sms);   // grid-stride loop: 32 CTAs per SM
  ProfScope prof("resize_linear_u8", (double)total * channels, (cudaStream_t)stream);
  resize_linear_u8_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint8_t *)src, (uint8_t *)dst, B, sh, sw, channels,
                                                                  dh, dw, scale_x, scale_y, area2);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

extern "C" int ctpn_image_blob_f32(const void *src_u8, const float *lut, int B, int sh, int sw, double fx, double fy, float *dst,
                                   int dh, int dw, void *stream) {
  CTPN_REQUIRE(src_u8 && lut && dst, "ctpn_image_blob_f32: null pointer");
  CTPN_REQUIRE(B > 0 && sh > 0 && sw > 0, "ctpn_image_blob_f32: bad shape");
  int eh = 0, ew = 0;
  int rc = ctpn_resize_out_size(sh, sw, fx, fy, &eh, &ew);
  if (rc) return rc;
  CTPN_REQUIRE(eh == dh && ew == dw, "ctpn_image_blob_f32: dst is %d x %d, cv2 would produce %d x %d", dh, dw, eh, ew);
  const double scale_x = 1.0 / fx, scale_y = 1.0 / fy;
  const int area2 = (scale_x == 2.0 && scale_y == 2.0) ? 1 : 0;
  const long long total = (long long)B * dh * dw;
  int sms = 0;
  if ((rc = current_sm_count(&sms))) return rc;
  const int grid = (int)std::min<long long>((total + 255) / 256, 32LL * sms);   // grid-stride loop: 32 CTAs per SM
  ProfScope prof("image_blob_f32", (double)total * 3, (cudaStream_t)stream);
  image_blob_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint8_t *)src_u8, lut, dst, B, sh, sw, dh, dw, scale_x,
                                                                scale_y, area2);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}
