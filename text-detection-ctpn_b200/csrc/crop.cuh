// The geometry of a text-line crop, ONE definition for the host widths (ctpn_line_crop_widths_host) and the crop kernels
// (ctpn_line_crops_u8, ctpn_line_crops_strided_u8, ctpn_line_crops_yuv420_u8: crop.cu).  A line is a row [x1,y1,x2,y2,x3,y3,x4,y4,score] of the connector's output, corners TL,
// TR, BL, BR; its crop of height hc is cv2.warpAffine of the resize_im output by the map below (oracle/crop.py):
//   len = sqrt((x2-x1)^2 + (y2-y1)^2), ht = sqrt((x3-x1)^2 + (y3-y1)^2), Wc = max(2, rint(hc * len / max(ht, 1)))
//   dst (0, 0) -> TL, (Wc-1, 0) -> TR, (0, hc-1) -> BL.
// float64 throughout, IEEE division and sqrt, and no FMA: g++ emits none for x86-64 and crop.cu is compiled with
// -fmad=false (csrc/Makefile), so host and device widths and maps agree bit for bit.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define CROP_HD __host__ __device__ __forceinline__
#else
#define CROP_HD inline
#endif

namespace ctpn {
namespace crop {

constexpr int kMinHeight = 2, kMaxHeight = 256;
constexpr int kMaxWidth = 1 << 20;     // a wider (or non-finite) width is refused, never allocated

// Wc of a line at crop height hc, or 0 when it is not finite or exceeds kMaxWidth
CROP_HD int width(const double *ln, int hc) {
  const double dx = ln[2] - ln[0], dy = ln[3] - ln[1], ex = ln[4] - ln[0], ey = ln[5] - ln[1];
  const double len = sqrt(dx * dx + dy * dy), ht = sqrt(ex * ex + ey * ey);
  const double w = rint((double)hc * len / (ht < 1.0 ? 1.0 : ht));   // max(ht, 1.0), first operand on NaN
  if (!(w <= (double)kMaxWidth)) return 0;                            // NaN, inf, too wide
  return w < 2.0 ? 2 : (int)w;
}

// Minv of a line of width wc (>= 2) at height hc: source point of destination pixel (x, y) is
// (m[0] x + m[1] y + m[2], m[3] x + m[4] y + m[5])
struct Map { double m[6]; };

CROP_HD Map map(const double *ln, int wc, int hc) {
  Map a;
  a.m[0] = (ln[2] - ln[0]) / (double)(wc - 1);
  a.m[1] = (ln[4] - ln[0]) / (double)(hc - 1);
  a.m[2] = ln[0];
  a.m[3] = (ln[3] - ln[1]) / (double)(wc - 1);
  a.m[4] = (ln[5] - ln[1]) / (double)(hc - 1);
  a.m[5] = ln[1];
  return a;
}

// The source line of a line of the resize_im frame at resize factor f: its corners divided by f, one IEEE float64 division
// each -- the division draw_boxes makes, and numpy's lines[:, :8] / f on the host, bit for bit.  Only TL, TR and BL
// (src[0..5]) enter the width and the map.
CROP_HD void source_line(const double *ln, double f, double *src) {
  for (int i = 0; i < 6; ++i) {
#ifdef __CUDA_ARCH__
    src[i] = __ddiv_rn(ln[i], f);
#else
    src[i] = ln[i] / f;
#endif
  }
}

}  // namespace crop
}  // namespace ctpn
