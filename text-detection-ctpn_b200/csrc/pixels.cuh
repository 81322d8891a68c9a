// Source images read in place, shared by the resize (resize.cu) and the line crops (crop.cu): the device accessors that
// give the sample (y, x, c) of a caller's image, and the host checks that fill them from a caller's descriptors.  An
// accessor gives the start of row y (row) and the sample at column x, channel c of such a row (at).
#pragma once
#include <limits.h>

#include <algorithm>

#include "common.cuh"

namespace ctpn {

// Anywhere, at signed byte strides per row, column and channel (a caller's device tensor read in place; a negative channel
// stride from channel 2 reads RGB as BGR, a zero stride broadcasts).
struct StridedPixels {
  const uint8_t *base;         // sample (0, 0, 0)
  long long row_stride;
  int col_stride, chan_stride;
  __device__ __forceinline__ const uint8_t *row(int y) const { return base + (long long)y * row_stride; }
  __device__ __forceinline__ uint8_t at(const uint8_t *r, int x, int c) const {
    return __ldg(r + ((long long)x * col_stride + (long long)c * chan_stride));
  }
};

// Converted from YUV 4:2:0 planes on the fly (video frames read in place), exactly as cv2.cvtColor(COLOR_YUV2BGR_NV12 /
// _NV21 / _I420 / _YV12) converts them: BT.601 limited range in 20-bit fixed point, nearest chroma -- chroma sample
// (y >> 1, x >> 1) serves luma sample (y, x).  Every term fits in int32 and >> is arithmetic, as in OpenCV's 4:2:0
// converters (restated and pinned against cv2 in oracle/yuv.py).  The row handle is a luma row plus the chroma rows of
// row >> 1; rows and columns come in clamped, so the chroma indices are in range too.
struct Yuv420Pixels {
  const uint8_t *y, *u, *v;    // sample (0, 0) of each plane
  long long y_row, u_row, v_row;
  int y_col, u_col, v_col;
  struct Row {
    const uint8_t *y, *u, *v;
  };
  __device__ __forceinline__ Row row(int r) const {
    return Row{y + (long long)r * y_row, u + (long long)(r >> 1) * u_row, v + (long long)(r >> 1) * v_row};
  }
  __device__ __forceinline__ uint8_t at(const Row &r, int x, int c) const {
    const int Y = __ldg(r.y + (long long)x * y_col);
    const int U = __ldg(r.u + (long long)(x >> 1) * u_col) - 128, V = __ldg(r.v + (long long)(x >> 1) * v_col) - 128;
    const int yy = max(Y - 16, 0) * 1220542 + (1 << 19);
    const int t = c == 0 ? yy + 2116026 * U : c == 1 ? yy - 852492 * V - 409993 * U : yy + 1673527 * V;
    return (uint8_t)min(max(t >> 20, 0), 255);
  }
};

// ---- host: a caller's descriptors -> an accessor, checked before any CUDA call ----------------------------------------------
// The lowest and the highest byte a box of extent[d] + 1 samples at byte strides st[d] touches, relative to the
// allocation, must lie in [0, bytes); 128-bit, so no stride can wrap them.  `what` names the box ("box", "Y plane").
static inline int box_in_allocation(const char *fn, int b, const char *what, long long off, const long long *st,
                                    const long long *extent, int dims, size_t bytes) {
  __int128 lo = off, hi = off;
  for (int d = 0; d < dims; ++d) {
    const __int128 span = (__int128)extent[d] * st[d];
    (span < 0 ? lo : hi) += span;
  }
  CTPN_REQUIRE(lo >= 0 && hi < (__int128)bytes, "%s: image %d: the %s spans bytes [%lld, %lld] of its allocation, outside [0, %zu)",
               fn, b, what, (long long)std::max<__int128>(std::min<__int128>(lo, LLONG_MAX), LLONG_MIN),
               (long long)std::max<__int128>(std::min<__int128>(hi, LLONG_MAX), LLONG_MIN), bytes);
  return CTPN_OK;
}

// Image b of a strided call: allocation src of src_bytes bytes, sample (0, 0, 0) at byte off, byte strides st[3] (row,
// column, channel), (sh, sw) pixels of 3 channels.  Refuses a NULL source, an empty size, column / channel strides outside
// 32 bits and a box outside the allocation.
static inline int strided_source(const char *fn, int b, const void *src, size_t src_bytes, long long off, const long long *st,
                                 int sh, int sw, StridedPixels *px) {
  CTPN_REQUIRE(src, "%s: image %d: null source", fn, b);
  CTPN_REQUIRE(sh > 0 && sw > 0, "%s: image %d: bad source size %d x %d", fn, b, sh, sw);
  CTPN_REQUIRE(st[1] >= INT_MIN && st[1] <= INT_MAX && st[2] >= INT_MIN && st[2] <= INT_MAX,
               "%s: image %d: column / channel stride (%lld, %lld) outside the 32-bit range", fn, b, st[1], st[2]);
  const long long extent[3] = {sh - 1, sw - 1, 2};
  const int rc = box_in_allocation(fn, b, "box", off, st, extent, 3, src_bytes);
  if (rc) return rc;
  *px = StridedPixels{(const uint8_t *)src + off, st[0], (int)st[1], (int)st[2]};
  return CTPN_OK;
}

// Frame b of a YUV 4:2:0 call: planes[3] (Y, U, V) of plane_bytes[3] bytes, sample (0, 0) at byte off[p], byte strides
// st[2p..2p+1] (row, column); Y is sh x sw, U and V sh/2 x sw/2.  Refuses odd or empty sides, a NULL plane, column strides
// outside 32 bits and a plane box outside its allocation, naming the plane.
static inline int yuv420_source(const char *fn, int b, const void *const *planes, const size_t *plane_bytes,
                                const long long *off, const long long *st, int sh, int sw, Yuv420Pixels *px) {
  static const char *const kPlane[3] = {"Y", "U", "V"}, *const kBox[3] = {"Y plane", "U plane", "V plane"};
  CTPN_REQUIRE(sh > 0 && sw > 0 && sh % 2 == 0 && sw % 2 == 0, "%s: image %d: source size %d x %d must be even and positive",
               fn, b, sh, sw);
  const uint8_t *p[3];
  for (int q = 0; q < 3; ++q) {
    const long long *s = st + 2 * q;
    CTPN_REQUIRE(planes[q], "%s: image %d: null %s plane", fn, b, kPlane[q]);
    CTPN_REQUIRE(s[1] >= INT_MIN && s[1] <= INT_MAX, "%s: image %d: %s plane column stride %lld outside the 32-bit range", fn,
                 b, kPlane[q], s[1]);
    const long long extent[2] = {(q ? sh / 2 : sh) - 1, (q ? sw / 2 : sw) - 1};
    const int rc = box_in_allocation(fn, b, kBox[q], off[q], s, extent, 2, plane_bytes[q]);
    if (rc) return rc;
    p[q] = (const uint8_t *)planes[q] + off[q];
  }
  *px = Yuv420Pixels{p[0], p[1], p[2], st[0], st[2], st[4], (int)st[1], (int)st[3], (int)st[5]};
  return CTPN_OK;
}

}  // namespace ctpn
