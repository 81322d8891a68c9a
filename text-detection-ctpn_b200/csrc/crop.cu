// Text-line crops on the device: cv2.warpAffine(image, Minv, (Wc, Hc), INTER_LINEAR | WARP_INVERSE_MAP, BORDER_REPLICATE)
// of every line of a batch (crop.cuh holds the width and the map, oracle/crop.py the recipe), cut out of
//   ctpn_line_crops_u8          the uint8 resize_im canvas the lines were found on, or
//   ctpn_line_crops_strided_u8  the source images at full resolution, read in place at any byte strides, by the source
//   ctpn_line_crops_yuv420_u8   lines lines / f (crop::source_line), or YUV 4:2:0 frames converted as cv2.cvtColor does.
// One CTA per (line, image); each thread computes output pixels in cv2's fixed point (crop_u8_pixel, shared by all three):
//   adelta = cvRound(m0 x 1024), X0 = cvRound((m1 y + m2) 1024) + 16, X = (X0 + adelta) >> 5   (likewise Y with m3..m5)
//   taps (X >> 5, Y >> 5) saturated to int16, each clamped to the image; fractions fx = X & 31, fy = Y & 31
//   dst = (32 (32-fx)(32-fy) p00 + 32 fx (32-fy) p01 + 32 (32-fx) fy p10 + 32 fx fy p11 + 16384) >> 15
// cvRound is round half to even (__double2int_rn).  This object is compiled with -fmad=false (csrc/Makefile), and the
// per-pixel products and sums use explicit _rn intrinsics besides, so that m1 y + m2 is never contracted.
#include <algorithm>

#include "common.cuh"
#include "crop.cuh"
#include "pixels.cuh"

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

// The canvas: image b's rows at row_pitch bytes, 3 interleaved BGR bytes per pixel
struct CanvasPixels {
  const unsigned char *im;
  int row_pitch;
  __device__ __forceinline__ const unsigned char *row(int y) const { return im + (size_t)y * row_pitch; }
  __device__ __forceinline__ unsigned char at(const unsigned char *r, int x, int c) const { return r[x * 3 + c]; }
};

// One output pixel (x, y) of the crop with map a out of an h x w image whose samples `src` gives -> o[3].  Taps, sat16,
// clamps, weights and rounding for every source kind, so the crop kernels agree by construction.
template <class Src>
__device__ __forceinline__ void crop_u8_pixel(const Src &src, int h, int w, const crop::Map &a, int x, int y,
                                              unsigned char *__restrict__ o) {
  const double xd = (double)x, yd = (double)y;
  const int adelta = __double2int_rn(__dmul_rn(__dmul_rn(a.m[0], xd), 1024.0));
  const int bdelta = __double2int_rn(__dmul_rn(__dmul_rn(a.m[3], xd), 1024.0));
  const long long x0 = (long long)__double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(a.m[1], yd), a.m[2]), 1024.0)) + 16;
  const long long y0 = (long long)__double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(a.m[4], yd), a.m[5]), 1024.0)) + 16;
  const long long X = (x0 + adelta) >> 5, Y = (y0 + bdelta) >> 5;
  const int sx = sat16(X >> 5), sy = sat16(Y >> 5), fx = (int)(X & 31), fy = (int)(Y & 31);
  const int c0 = clampi(sx, 0, w - 1), c1 = clampi(sx + 1, 0, w - 1);
  const auto r0 = src.row(clampi(sy, 0, h - 1)), r1 = src.row(clampi(sy + 1, 0, h - 1));
  const int w00 = 32 * (32 - fx) * (32 - fy), w01 = 32 * fx * (32 - fy), w10 = 32 * (32 - fx) * fy, w11 = 32 * fx * fy;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int v = (src.at(r0, c0, c) * w00 + src.at(r0, c1, c) * w01 + src.at(r1, c0, c) * w10 + src.at(r1, c1, c) * w11 +
                   16384) >> 15;
    o[c] = (unsigned char)(v > 255 ? 255 : v);
  }
}

// The CTA's line ln (TL, TR, BL in ln[0..5], in the frame of the image `src` gives) into dst [hc][wmax][3], zeros past its
// width; a width that is not the one the caller sized the output by writes nothing and sets *status.
template <class Src>
__device__ __forceinline__ void crop_line(const Src &src, int h, int w, const double *ln, int hc, int wmax,
                                          unsigned char *__restrict__ dst, int *__restrict__ status) {
  const int wc = crop::width(ln, hc);
  if (wc == 0 || wc > wmax) {
    if (threadIdx.x == 0) *status = 1;
    return;
  }
  const crop::Map a = crop::map(ln, wc, hc);
  const int n = hc * wmax;
  for (int i = threadIdx.x; i < n; i += kCropThreads) {
    const int y = i / wmax, x = i - y * wmax;
    unsigned char *o = dst + (size_t)i * 3;
    if (x >= wc) {
      o[0] = o[1] = o[2] = 0;
      continue;
    }
    crop_u8_pixel(src, h, w, a, x, y, o);
  }
}

__global__ void __launch_bounds__(kCropThreads)
line_crops_kernel(const unsigned char *__restrict__ canvas, long long batch_pitch, int row_pitch,
                  const double *__restrict__ lines, int rows, int hc, const __grid_constant__ CropBatch p,
                  int *__restrict__ status) {
  const int j = blockIdx.x, b = blockIdx.y;
  if (j >= p.m[b]) return;
  crop_line(CanvasPixels{canvas + (size_t)b * batch_pitch, row_pitch}, p.h[b], p.w[b], lines + ((size_t)b * rows + j) * 9,
            hc, p.wmax[b], p.out[b] + (size_t)j * hc * p.wmax[b] * 3, status + b);
}

// ---- crops out of the source images: the lines divided by f, the sources read in place ----------------------------------
// Strided sources (host images uploaded whole, CUDA tensors): 56 bytes per image, 64 images in one launch.
struct StridedCropBatch {
  const uint8_t *base[kCropMaxBatch];  // sample (0, 0, 0) of image b
  long long row_stride[kCropMaxBatch];
  unsigned char *out[kCropMaxBatch];   // [m][hc][wmax][3] per image
  double f[kCropMaxBatch];             // resize_im factor: source line = line / f
  int col_stride[kCropMaxBatch], chan_stride[kCropMaxBatch];
  int m[kCropMaxBatch], wmax[kCropMaxBatch], h[kCropMaxBatch], w[kCropMaxBatch];
};
// YUV 4:2:0 frames: three planes take 92 bytes per frame, so a launch takes kCropYuvChunk of them.
constexpr int kCropYuvChunk = 32;
struct Yuv420CropBatch {
  const uint8_t *plane[kCropYuvChunk][3];  // sample (0, 0) of the Y, U and V plane of frame b
  long long row_stride[kCropYuvChunk][3];
  unsigned char *out[kCropYuvChunk];
  double f[kCropYuvChunk];
  int col_stride[kCropYuvChunk][3];
  int m[kCropYuvChunk], wmax[kCropYuvChunk], h[kCropYuvChunk], w[kCropYuvChunk];
};
// the other parameters of a source-crop kernel: lines, rows, hc, status
constexpr size_t kSourceCropArgs = sizeof(double *) + 2 * sizeof(int) + sizeof(int *);
static_assert(sizeof(StridedCropBatch) == 56 * kCropMaxBatch, "56 bytes per strided source");
static_assert(sizeof(Yuv420CropBatch) == 92 * kCropYuvChunk, "92 bytes per YUV 4:2:0 source");
static_assert(sizeof(StridedCropBatch) + kSourceCropArgs <= 4096, "strided crop parameters exceed 4 KB");
static_assert(sizeof(Yuv420CropBatch) + kSourceCropArgs <= 4096, "yuv420 crop parameters exceed 4 KB");

__global__ void __launch_bounds__(kCropThreads)
line_crops_strided_kernel(const double *__restrict__ lines, int rows, int hc, const __grid_constant__ StridedCropBatch p,
                          int *__restrict__ status) {
  const int j = blockIdx.x, b = blockIdx.y;
  if (j >= p.m[b]) return;
  double ln[6];
  crop::source_line(lines + ((size_t)b * rows + j) * 9, p.f[b], ln);
  crop_line(StridedPixels{p.base[b], p.row_stride[b], p.col_stride[b], p.chan_stride[b]}, p.h[b], p.w[b], ln, hc, p.wmax[b],
            p.out[b] + (size_t)j * hc * p.wmax[b] * 3, status + b);
}

// lines and status start at the chunk's first frame
__global__ void __launch_bounds__(kCropThreads)
line_crops_yuv420_kernel(const double *__restrict__ lines, int rows, int hc, const __grid_constant__ Yuv420CropBatch p,
                         int *__restrict__ status) {
  const int j = blockIdx.x, b = blockIdx.y;
  if (j >= p.m[b]) return;
  double ln[6];
  crop::source_line(lines + ((size_t)b * rows + j) * 9, p.f[b], ln);
  const Yuv420Pixels src{p.plane[b][0], p.plane[b][1], p.plane[b][2], p.row_stride[b][0], p.row_stride[b][1],
                         p.row_stride[b][2], p.col_stride[b][0], p.col_stride[b][1], p.col_stride[b][2]};
  crop_line(src, p.h[b], p.w[b], ln, hc, p.wmax[b], p.out[b] + (size_t)j * hc * p.wmax[b] * 3, status + b);
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

// The per-image output rules of the source-crop entries: 0 <= m <= rows, a finite f > 0, and where m > 0 an output and a
// padded width 2..kMaxWidth.
static int source_crop_image_ok(const char *fn, int b, int m, int rows, double f, const void *out, int wm) {
  CTPN_REQUIRE(m >= 0 && m <= rows, "%s: image %d: %d lines, must be 0..rows = %d", fn, b, m, rows);
  CTPN_REQUIRE(f > 0.0 && f <= 1.7976931348623157e308, "%s: image %d: resize factor %g, must be finite and > 0", fn, b, f);
  if (m > 0) {
    CTPN_REQUIRE(out, "%s: image %d: null output with %d lines", fn, b, m);
    CTPN_REQUIRE(wm >= 2 && wm <= crop::kMaxWidth, "%s: image %d: padded width %d, must be 2..%d", fn, b, wm, crop::kMaxWidth);
  }
  return CTPN_OK;
}

static int source_crop_call_ok(const char *fn, int batch, int rows, int hc) {
  CTPN_REQUIRE(batch >= 1 && batch <= kCropMaxBatch, "%s: batch = %d, must be 1..%d", fn, batch, kCropMaxBatch);
  CTPN_REQUIRE(hc >= crop::kMinHeight && hc <= crop::kMaxHeight, "%s: crop height %d, must be %d..%d", fn, hc,
               crop::kMinHeight, crop::kMaxHeight);
  CTPN_REQUIRE(rows >= 0, "%s: rows = %d, must be >= 0", fn, rows);
  return CTPN_OK;
}

extern "C" int ctpn_line_crops_strided_u8(const void *const *src, const size_t *src_bytes, const long long *src_offset,
                                          const long long *src_strides, const int *src_hw, const double *f, const double *lines,
                                          int batch, int rows, int hc, const int *num_lines, const int *max_width,
                                          void *const *out, int *status, void *stream) {
  const char *fn = "ctpn_line_crops_strided_u8";
  CTPN_REQUIRE(src && src_bytes && src_offset && src_strides && src_hw && f && num_lines && max_width && out,
               "%s: null descriptor array", fn);
  int rc = source_crop_call_ok(fn, batch, rows, hc);
  if (rc) return rc;
  StridedCropBatch p;
  memset(&p, 0, sizeof(p));
  int max_m = 0;
  double work = 0.0;
  for (int b = 0; b < batch; ++b) {
    const int m = num_lines[b], wm = max_width[b];
    if ((rc = source_crop_image_ok(fn, b, m, rows, f[b], out[b], wm))) return rc;
    StridedPixels px;
    if ((rc = strided_source(fn, b, src[b], src_bytes[b], src_offset[b], src_strides + 3 * b, src_hw[2 * b], src_hw[2 * b + 1],
                             &px)))
      return rc;
    p.base[b] = px.base;
    p.row_stride[b] = px.row_stride;
    p.col_stride[b] = px.col_stride;
    p.chan_stride[b] = px.chan_stride;
    p.out[b] = (unsigned char *)out[b];
    p.f[b] = f[b];
    p.m[b] = m;
    p.wmax[b] = wm;
    p.h[b] = src_hw[2 * b];
    p.w[b] = src_hw[2 * b + 1];
    max_m = std::max(max_m, m);
    work += (double)m * hc * wm * 3;
  }
  CTPN_REQUIRE(max_m == 0 || (lines && status), "%s: null lines or status", fn);
  int sms = 0;
  if ((rc = current_sm_count(&sms))) return rc;        // also CTPN_ERR_NO_DEVICE without a GPU
  if (max_m == 0) return CTPN_OK;
  ProfScope prof("line_crops_strided_u8", work, (cudaStream_t)stream);
  line_crops_strided_kernel<<<dim3((unsigned)max_m, (unsigned)batch), kCropThreads, 0, (cudaStream_t)stream>>>(lines, rows, hc, p,
                                                                                                              status);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

extern "C" int ctpn_line_crops_yuv420_u8(const void *const *planes, const size_t *plane_bytes, const long long *plane_offset,
                                         const long long *plane_strides, const int *src_hw, const double *f, const double *lines,
                                         int batch, int rows, int hc, const int *num_lines, const int *max_width,
                                         void *const *out, int *status, void *stream) {
  const char *fn = "ctpn_line_crops_yuv420_u8";
  CTPN_REQUIRE(planes && plane_bytes && plane_offset && plane_strides && src_hw && f && num_lines && max_width && out,
               "%s: null descriptor array", fn);
  int rc = source_crop_call_ok(fn, batch, rows, hc);
  if (rc) return rc;
  constexpr int kChunks = (kCropMaxBatch + kCropYuvChunk - 1) / kCropYuvChunk;
  Yuv420CropBatch chunk[kChunks];
  memset(chunk, 0, sizeof(chunk));
  int max_m[kChunks] = {};
  double work = 0.0;
  for (int b = 0; b < batch; ++b) {
    const int m = num_lines[b], wm = max_width[b];
    if ((rc = source_crop_image_ok(fn, b, m, rows, f[b], out[b], wm))) return rc;
    Yuv420Pixels px;
    if ((rc = yuv420_source(fn, b, planes + 3 * b, plane_bytes + 3 * b, plane_offset + 3 * b, plane_strides + 6 * b,
                            src_hw[2 * b], src_hw[2 * b + 1], &px)))
      return rc;
    Yuv420CropBatch &p = chunk[b / kCropYuvChunk];
    const int k = b % kCropYuvChunk;
    const uint8_t *const pl[3] = {px.y, px.u, px.v};
    const long long rs[3] = {px.y_row, px.u_row, px.v_row};
    const int cs[3] = {px.y_col, px.u_col, px.v_col};
    for (int q = 0; q < 3; ++q) {
      p.plane[k][q] = pl[q];
      p.row_stride[k][q] = rs[q];
      p.col_stride[k][q] = cs[q];
    }
    p.out[k] = (unsigned char *)out[b];
    p.f[k] = f[b];
    p.m[k] = m;
    p.wmax[k] = wm;
    p.h[k] = src_hw[2 * b];
    p.w[k] = src_hw[2 * b + 1];
    max_m[b / kCropYuvChunk] = std::max(max_m[b / kCropYuvChunk], m);
    work += (double)m * hc * wm * 3;
  }
  CTPN_REQUIRE(*std::max_element(max_m, max_m + kChunks) == 0 || (lines && status), "%s: null lines or status", fn);
  int sms = 0;
  if ((rc = current_sm_count(&sms))) return rc;        // also CTPN_ERR_NO_DEVICE without a GPU
  ProfScope prof("line_crops_yuv420_u8", work, (cudaStream_t)stream);
  for (int first = 0; first < batch; first += kCropYuvChunk) {
    const int nb = std::min(kCropYuvChunk, batch - first), c = first / kCropYuvChunk;
    if (max_m[c] == 0) continue;
    line_crops_yuv420_kernel<<<dim3((unsigned)max_m[c], (unsigned)nb), kCropThreads, 0, (cudaStream_t)stream>>>(
        lines + (size_t)first * rows * 9, rows, hc, chunk[c], status + first);
    CTPN_LAUNCH_CHECK();
  }
  return CTPN_OK;
}
