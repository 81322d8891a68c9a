// Text-line crops on the device: cv2.warpAffine(resized, Minv, (Wc, Hc), INTER_LINEAR | WARP_INVERSE_MAP,
// BORDER_REPLICATE) of every line of a batch, out of the uint8 resize_im canvas the lines were found on (crop.cuh holds
// the width and the map, oracle/crop.py the recipe).  One CTA per (line, image); each thread computes output pixels in
// cv2's fixed point:
//   adelta = cvRound(m0 x 1024), X0 = cvRound((m1 y + m2) 1024) + 16, X = (X0 + adelta) >> 5   (likewise Y with m3..m5)
//   taps (X >> 5, Y >> 5) saturated to int16, each clamped to the image; fractions fx = X & 31, fy = Y & 31
//   dst = (32 (32-fx)(32-fy) p00 + 32 fx (32-fy) p01 + 32 (32-fx) fy p10 + 32 fx fy p11 + 16384) >> 15
// cvRound is round half to even (__double2int_rn).  This object is compiled with -fmad=false (csrc/Makefile), and the
// per-pixel products and sums use explicit _rn intrinsics besides, so that m1 y + m2 is never contracted.
#include <algorithm>

#include "common.cuh"
#include "crop.cuh"

namespace ctpn {
namespace {

constexpr int kCropMaxBatch = 64;
constexpr int kCropThreads = 128;

// per-image descriptors, passed by value (1.5 KB of the 4 KB parameter space)
struct CropBatch {
  unsigned char *out[kCropMaxBatch];   // [m][hc][wmax][3] per image
  int m[kCropMaxBatch], wmax[kCropMaxBatch], h[kCropMaxBatch], w[kCropMaxBatch];
};

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

__device__ __forceinline__ int sat16(long long v) { return v < -32768 ? -32768 : (v > 32767 ? 32767 : (int)v); }

__global__ void __launch_bounds__(kCropThreads)
line_crops_kernel(const unsigned char *__restrict__ canvas, long long batch_pitch, int row_pitch,
                  const double *__restrict__ lines, int rows, int hc, const __grid_constant__ CropBatch p,
                  int *__restrict__ status) {
  const int j = blockIdx.x, b = blockIdx.y;
  if (j >= p.m[b]) return;
  const double *ln = lines + ((size_t)b * rows + j) * 9;
  const int wmax = p.wmax[b];
  const int wc = crop::width(ln, hc);
  if (wc == 0 || wc > wmax) {                          // not the width the caller sized the output by: write nothing
    if (threadIdx.x == 0) status[b] = 1;
    return;
  }
  const crop::Map a = crop::map(ln, wc, hc);
  const int h = p.h[b], w = p.w[b];
  const unsigned char *src = canvas + (size_t)b * batch_pitch;
  unsigned char *dst = p.out[b] + (size_t)j * hc * wmax * 3;
  const int n = hc * wmax;
  for (int i = threadIdx.x; i < n; i += kCropThreads) {
    const int y = i / wmax, x = i - y * wmax;
    unsigned char *o = dst + (size_t)i * 3;
    if (x >= wc) {
      o[0] = o[1] = o[2] = 0;
      continue;
    }
    const double xd = (double)x, yd = (double)y;
    const int adelta = __double2int_rn(__dmul_rn(__dmul_rn(a.m[0], xd), 1024.0));
    const int bdelta = __double2int_rn(__dmul_rn(__dmul_rn(a.m[3], xd), 1024.0));
    const long long x0 = (long long)__double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(a.m[1], yd), a.m[2]), 1024.0)) + 16;
    const long long y0 = (long long)__double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(a.m[4], yd), a.m[5]), 1024.0)) + 16;
    const long long X = (x0 + adelta) >> 5, Y = (y0 + bdelta) >> 5;
    const int sx = sat16(X >> 5), sy = sat16(Y >> 5), fx = (int)(X & 31), fy = (int)(Y & 31);
    const int c0 = clampi(sx, 0, w - 1) * 3, c1 = clampi(sx + 1, 0, w - 1) * 3;
    const unsigned char *r0 = src + (size_t)clampi(sy, 0, h - 1) * row_pitch;
    const unsigned char *r1 = src + (size_t)clampi(sy + 1, 0, h - 1) * row_pitch;
    const int w00 = 32 * (32 - fx) * (32 - fy), w01 = 32 * fx * (32 - fy), w10 = 32 * (32 - fx) * fy, w11 = 32 * fx * fy;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int v = (r0[c0 + c] * w00 + r0[c1 + c] * w01 + r1[c0 + c] * w10 + r1[c1 + c] * w11 + 16384) >> 15;
      o[c] = (unsigned char)(v > 255 ? 255 : v);
    }
  }
}

}  // namespace
}  // namespace ctpn

using namespace ctpn;

extern "C" int ctpn_line_crop_widths_host(const double *lines, int n, int hc, int *widths) {
  CTPN_REQUIRE(n >= 0, "ctpn_line_crop_widths_host: n = %d, must be >= 0", n);
  CTPN_REQUIRE(n == 0 || (lines && widths), "ctpn_line_crop_widths_host: null pointer");
  CTPN_REQUIRE(hc >= crop::kMinHeight && hc <= crop::kMaxHeight, "ctpn_line_crop_widths_host: crop height %d, must be %d..%d",
               hc, crop::kMinHeight, crop::kMaxHeight);
  for (int j = 0; j < n; ++j) {
    const int wc = crop::width(lines + (size_t)j * 9, hc);
    CTPN_REQUIRE(wc > 0, "ctpn_line_crop_widths_host: line %d: its crop width is not finite or exceeds %d", j,
                 crop::kMaxWidth);
    widths[j] = wc;
  }
  return CTPN_OK;
}

extern "C" int ctpn_line_crops_u8(const void *canvas, long long batch_pitch, int row_pitch, const int *im_hw, const double *lines,
                                  int batch, int rows, int hc, const int *num_lines, const int *max_width, void *const *out,
                                  int *status, void *stream) {
  const char *fn = "ctpn_line_crops_u8";
  CTPN_REQUIRE(im_hw && num_lines && max_width && out, "%s: null descriptor array", fn);
  CTPN_REQUIRE(batch >= 1 && batch <= kCropMaxBatch, "%s: batch = %d, must be 1..%d", fn, batch, kCropMaxBatch);
  CTPN_REQUIRE(hc >= crop::kMinHeight && hc <= crop::kMaxHeight, "%s: crop height %d, must be %d..%d", fn, hc,
               crop::kMinHeight, crop::kMaxHeight);
  CTPN_REQUIRE(rows >= 0, "%s: rows = %d, must be >= 0", fn, rows);
  CTPN_REQUIRE(row_pitch > 0 && batch_pitch > 0, "%s: bad canvas pitches %lld / %d", fn, batch_pitch, row_pitch);
  CropBatch p;
  memset(&p, 0, sizeof(p));
  int max_m = 0;
  double work = 0.0;
  for (int b = 0; b < batch; ++b) {
    const int h = im_hw[2 * b], w = im_hw[2 * b + 1], m = num_lines[b], wm = max_width[b];
    CTPN_REQUIRE(m >= 0 && m <= rows, "%s: image %d: %d lines, must be 0..rows = %d", fn, b, m, rows);
    CTPN_REQUIRE(h >= 1 && w >= 1, "%s: image %d: bad size %d x %d", fn, b, h, w);
    CTPN_REQUIRE((long long)w * 3 <= row_pitch && (long long)h * row_pitch <= batch_pitch,
                 "%s: image %d: %d x %d x 3 does not fit the canvas pitches (row %d, image %lld bytes)", fn, b, h, w, row_pitch,
                 batch_pitch);
    if (m > 0) {
      CTPN_REQUIRE(out[b], "%s: image %d: null output with %d lines", fn, b, m);
      CTPN_REQUIRE(wm >= 2 && wm <= crop::kMaxWidth, "%s: image %d: padded width %d, must be 2..%d", fn, b, wm,
                   crop::kMaxWidth);
    }
    p.out[b] = (unsigned char *)out[b];
    p.m[b] = m;
    p.wmax[b] = wm;
    p.h[b] = h;
    p.w[b] = w;
    max_m = std::max(max_m, m);
    work += (double)m * hc * wm * 3;
  }
  CTPN_REQUIRE(max_m == 0 || (canvas && lines && status), "%s: null canvas, lines or status", fn);
  int sms = 0, rc;
  if ((rc = current_sm_count(&sms))) return rc;        // also CTPN_ERR_NO_DEVICE without a GPU
  if (max_m == 0) return CTPN_OK;
  ProfScope prof("line_crops_u8", work, (cudaStream_t)stream);
  line_crops_kernel<<<dim3((unsigned)max_m, (unsigned)batch), kCropThreads, 0, (cudaStream_t)stream>>>(
      (const unsigned char *)canvas, batch_pitch, row_pitch, lines, rows, hc, p, status);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}
