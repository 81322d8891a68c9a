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
//
// The *_ragged entry points run both for a batch of images of different sizes (Engine.rois_images); they share the
// per-pixel functions below with the single-image kernels.  ctpn_resize_linear_u8_ragged_rows is the ragged resize on
// sources that hold only the rows it reads (Engine.stream_rois_images uploads camera photos that way), and
// ctpn_resize_linear_u8_strided the ragged resize on images read in place at any byte strides (CUDA tensors of callers);
// ctpn_resize_linear_u8_yuv420 converts YUV 4:2:0 frames read in place to BGR as cv2.cvtColor does, inside that resize.
#include "common.cuh"
#include "pixels.cuh"

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

// Where sample (y, x, c) of a source image is stored.  An accessor gives the start of row y (row) and the sample at
// column x, channel c of such a row (at).  Interleaved [h][pitch][C] images with every row in place ...
struct DenseRows {
  const uint8_t *__restrict__ im;
  int pitch, C;
  __device__ __forceinline__ const uint8_t *row(int y) const { return im + (size_t)y * pitch * C; }
  __device__ __forceinline__ uint8_t at(const uint8_t *r, int x, int c) const { return r[(size_t)x * C + c]; }
};
// ... or only the rows the resize reads (ctpn_resize_linear_u8_ragged_rows): map[y] is the stored index of source row y.
// The map is device memory the host never saw, so the index is clamped to the stored extent the host did check.
struct CompactRows {
  const uint8_t *__restrict__ im;
  int pitch, C;
  const int *__restrict__ map;
  int stored;
  __device__ __forceinline__ const uint8_t *row(int y) const {
    return im + (size_t)min(max(__ldg(map + y), 0), stored - 1) * pitch * C;
  }
  __device__ __forceinline__ uint8_t at(const uint8_t *r, int x, int c) const { return r[(size_t)x * C + c]; }
};
// ... or anywhere, at signed byte strides (StridedPixels: ctpn_resize_linear_u8_strided), or converted from YUV 4:2:0
// planes on the fly (Yuv420Pixels: ctpn_resize_linear_u8_yuv420) -- pixels.cuh, shared with the line crops.

// One output pixel of cv2.resize(INTER_LINEAR) of a uint8 image of sh x sw pixels and C channels -> o[C].  Shared by
// every uint8 resize kernel: a ragged or strided batch is bit-identical to single-image runs by construction.  Taps,
// weights, the INTER_AREA route and rounding come from the source geometry (sh, sw); only the value of a sample comes from
// the accessor `src`, whose row handle is whatever its row() returns.
template <class Src>
__device__ __forceinline__ void resize_u8_pixel(const Src src, int sh, int sw, int C, int dx, int dy, double scale_x,
                                                double scale_y, bool area2, uint8_t *__restrict__ o) {
  if (area2) {
    const int y0 = 2 * dy, x0 = 2 * dx;
    const int ny = min(2, sh - y0), nx = min(2, sw - x0);
    for (int c = 0; c < C; ++c) {
      int sum = 0;
      for (int yy = 0; yy < ny; ++yy) {
        const auto r = src.row(y0 + yy);
        for (int xx = 0; xx < nx; ++xx) sum += src.at(r, x0 + xx, c);
      }
      int v = (ny * nx == 4) ? (sum + 2) >> 2 : __float2int_rn(__fdiv_rn((float)sum, (float)(ny * nx)));
      o[c] = (uint8_t)min(max(v, 0), 255);
    }
    return;
  }
  int sx0, sx1, a0, a1, sy0, sy1, b0, b1;
  resize_taps(dx, sw, scale_x, true, sx0, sx1, a0, a1);
  resize_taps(dy, sh, scale_y, false, sy0, sy1, b0, b1);
  const auto r0 = src.row(sy0), r1 = src.row(sy1);
  for (int c = 0; c < C; ++c) {
    const int h0 = src.at(r0, sx0, c) * a0 + src.at(r0, sx1, c) * a1;
    const int h1 = src.at(r1, sx0, c) * a0 + src.at(r1, sx1, c) * a1;
    const int v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
    o[c] = (uint8_t)min(max(v, 0), 255);
  }
}

__global__ void __launch_bounds__(256)
resize_linear_u8_kernel(const uint8_t *__restrict__ src, uint8_t *__restrict__ dst, int B, int sh, int sw, int C, int dh,
                        int dw, double scale_x, double scale_y, int area2) {
  const long long total = (long long)B * dh * dw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int dx = (int)(i % dw), dy = (int)((i / dw) % dh), b = (int)(i / ((long long)dw * dh));
    resize_u8_pixel(DenseRows{src + (size_t)b * sh * sw * C, sw, C}, sh, sw, C, dx, dy, scale_x, scale_y, area2 != 0,
                    dst + (size_t)i * C);
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

// One output pixel of the mean-subtracted float32 blob of a uint8 BGR image im [sh][pitch][3] at another scale -> o[3]
// (lut[256][3] = float32(double(v) - mean[c])).  Shared by the uniform and the ragged kernel.
__device__ __forceinline__ void image_blob_pixel(const uint8_t *__restrict__ im, int sh, int sw, int pitch,
                                                 const float *__restrict__ lut, int dx, int dy, double scale_x, double scale_y,
                                                 bool area2, float *__restrict__ o) {
  auto px = [&](int y, int x, int c) { return __ldg(lut + im[((size_t)y * pitch + x) * 3 + c] * 3 + c); };
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
    return;
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

// uint8 BGR image -> mean-subtracted float32 blob at another scale (3 channels)
__global__ void __launch_bounds__(256)
image_blob_f32_kernel(const uint8_t *__restrict__ src, const float *__restrict__ lut, float *__restrict__ dst, int B, int sh,
                      int sw, int dh, int dw, double scale_x, double scale_y, int area2) {
  const long long total = (long long)B * dh * dw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int dx = (int)(i % dw), dy = (int)((i / dw) % dh), b = (int)(i / ((long long)dw * dh));
    image_blob_pixel(src + (size_t)b * sh * sw * 3, sh, sw, sw, lut, dx, dy, scale_x, scale_y, area2 != 0, dst + (size_t)i * 3);
  }
}

// ---- ragged batches: image b has its own source (offset, h, w, row pitch), scale and output size; its output goes to
// rows < dh[b], columns < dw[b] of slice b of the canvas [B][H][W][C], the rest of the canvas is not written.  The host
// validates every descriptor and passes them by value (one __grid_constant__ struct, read in place from the parameter
// bank), so a kernel only touches memory whose extent the host checked.  grid.y = image: after resize_im the outputs
// of one batch differ in area by about 2x, so equal x-extents per image balance well.
constexpr int kRaggedMax = 64;
struct RaggedResize {
  long long src_offset[kRaggedMax];    // elements (bytes) from the source base to pixel (0, 0) of image b
  double scale_x[kRaggedMax], scale_y[kRaggedMax];
  int sh[kRaggedMax], sw[kRaggedMax], pitch[kRaggedMax], dh[kRaggedMax], dw[kRaggedMax];
  unsigned long long area2;            // bit b: exact 1/2 in both directions (INTER_AREA routing of cv::resize)
  int H, W, C;
};

__global__ void __launch_bounds__(256) resize_linear_u8_ragged_kernel(const uint8_t *__restrict__ src, uint8_t *__restrict__ dst,
                                                                      const __grid_constant__ RaggedResize p) {
  const int b = blockIdx.y, dh = p.dh[b], dw = p.dw[b], C = p.C;
  const uint8_t *im = src + p.src_offset[b];
  uint8_t *out = dst + (size_t)b * p.H * p.W * C;
  const long long total = (long long)dh * dw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int dx = (int)(i % dw), dy = (int)(i / dw);
    resize_u8_pixel(DenseRows{im, p.pitch[b], C}, p.sh[b], p.sw[b], C, dx, dy, p.scale_x[b], p.scale_y[b], (p.area2 >> b) & 1,
                    out + ((size_t)dy * p.W + dx) * C);
  }
}

// Row-compacted sources: image b stores only stored[b] of its sh[b] rows, and rows + map_offset[b] is its row map
// (sh[b] entries, see CompactRows).  Same launch shape and per-pixel code as the kernel above.
struct RaggedResizeRows {
  RaggedResize r;
  long long map_offset[kRaggedMax];
  int stored[kRaggedMax];
};

__global__ void __launch_bounds__(256) resize_linear_u8_ragged_rows_kernel(const uint8_t *__restrict__ src,
                                                                           const int *__restrict__ rows, uint8_t *__restrict__ dst,
                                                                           const __grid_constant__ RaggedResizeRows q) {
  const RaggedResize &p = q.r;
  const int b = blockIdx.y, dh = p.dh[b], dw = p.dw[b], C = p.C;
  const uint8_t *im = src + p.src_offset[b];
  const CompactRows src_b{im, p.pitch[b], C, rows + q.map_offset[b], q.stored[b]};
  uint8_t *out = dst + (size_t)b * p.H * p.W * C;
  const long long total = (long long)dh * dw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int dx = (int)(i % dw), dy = (int)(i / dw);
    resize_u8_pixel(src_b, p.sh[b], p.sw[b], C, dx, dy, p.scale_x[b], p.scale_y[b], (p.area2 >> b) & 1,
                    out + ((size_t)dy * p.W + dx) * C);
  }
}

// Images read in place at byte strides of their own (ctpn_resize_linear_u8_strided), written as the dense ragged kernel
// writes them: 3 channels, canvas [B][H][W][3].  56 bytes per image, 3600 in all: with the dst pointer the kernel's
// parameters stay within the 4 KB every CUDA 12 driver accepts, so the column and channel strides are 32-bit (the host
// checks that they fit).
struct StridedResize {
  const uint8_t *base[kRaggedMax];     // sample (0, 0, 0) of image b
  long long row_stride[kRaggedMax];
  int col_stride[kRaggedMax], chan_stride[kRaggedMax];
  double scale_x[kRaggedMax], scale_y[kRaggedMax];
  int sh[kRaggedMax], sw[kRaggedMax], dh[kRaggedMax], dw[kRaggedMax];
  unsigned long long area2;            // bit b: exact 1/2 in both directions
  int H, W;
};
static_assert(sizeof(StridedResize) + sizeof(void *) <= 4096, "strided resize parameters exceed 4 KB");

__global__ void __launch_bounds__(256) resize_linear_u8_strided_kernel(uint8_t *__restrict__ dst,
                                                                       const __grid_constant__ StridedResize p) {
  const int b = blockIdx.y, dh = p.dh[b], dw = p.dw[b];
  const StridedPixels src_b{p.base[b], p.row_stride[b], p.col_stride[b], p.chan_stride[b]};
  uint8_t *out = dst + (size_t)b * p.H * p.W * 3;
  const long long total = (long long)dh * dw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int dx = (int)(i % dw), dy = (int)(i / dw);
    resize_u8_pixel(src_b, p.sh[b], p.sw[b], 3, dx, dy, p.scale_x[b], p.scale_y[b], (p.area2 >> b) & 1,
                    out + ((size_t)dy * p.W + dx) * 3);
  }
}

// YUV 4:2:0 frames read in place (ctpn_resize_linear_u8_yuv420), written as the strided kernel writes them.  Three planes
// per image take 92 bytes of descriptors, so 64 images (5.9 KB) would exceed the 4 KB of kernel parameters; the host
// launches chunks of up to kYuvChunk images, each writing its own canvas slices.
constexpr int kYuvChunk = 32;
struct Yuv420Resize {
  const uint8_t *plane[kYuvChunk][3];  // sample (0, 0) of the Y, U and V plane of image b
  long long row_stride[kYuvChunk][3];
  int col_stride[kYuvChunk][3];
  double scale_x[kYuvChunk], scale_y[kYuvChunk];
  int sh[kYuvChunk], sw[kYuvChunk], dh[kYuvChunk], dw[kYuvChunk];
  unsigned area2;                      // bit b: exact 1/2 in both directions
  int H, W;
};
static_assert(sizeof(Yuv420Resize) + sizeof(void *) <= 4096, "yuv420 resize parameters exceed 4 KB");

__global__ void __launch_bounds__(256) resize_linear_u8_yuv420_kernel(uint8_t *__restrict__ dst,
                                                                      const __grid_constant__ Yuv420Resize p) {
  const int b = blockIdx.y, dh = p.dh[b], dw = p.dw[b];
  const Yuv420Pixels src_b{p.plane[b][0], p.plane[b][1], p.plane[b][2],
                           p.row_stride[b][0], p.row_stride[b][1], p.row_stride[b][2],
                           p.col_stride[b][0], p.col_stride[b][1], p.col_stride[b][2]};
  uint8_t *out = dst + (size_t)b * p.H * p.W * 3;
  const long long total = (long long)dh * dw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int dx = (int)(i % dw), dy = (int)(i / dw);
    resize_u8_pixel(src_b, p.sh[b], p.sw[b], 3, dx, dy, p.scale_x[b], p.scale_y[b], (p.area2 >> b) & 1,
                    out + ((size_t)dy * p.W + dx) * 3);
  }
}

__global__ void __launch_bounds__(256) image_blob_f32_ragged_kernel(const uint8_t *__restrict__ src, const float *__restrict__ lut,
                                                                    float *__restrict__ dst, const __grid_constant__ RaggedResize p) {
  const int b = blockIdx.y, dh = p.dh[b], dw = p.dw[b];
  const uint8_t *im = src + p.src_offset[b];
  float *out = dst + (size_t)b * p.H * p.W * 3;
  const long long total = (long long)dh * dw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int dx = (int)(i % dw), dy = (int)(i / dw);
    image_blob_pixel(im, p.sh[b], p.sw[b], p.pitch[b], lut, dx, dy, p.scale_x[b], p.scale_y[b], (p.area2 >> b) & 1,
                     out + ((size_t)dy * p.W + dx) * 3);
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

// The per-image geometry rules of every ragged call: source size and scales, then the output size cv2 would produce,
// which dst_hw must give and the canvas must hold.
static int ragged_geometry_ok(const char *fn, int b, int sh, int sw, double fx, double fy, const int *dst_hw, int H, int W,
                              int *eh, int *ew) {
  CTPN_REQUIRE(sh > 0 && sw > 0, "%s: image %d: bad source size %d x %d", fn, b, sh, sw);
  CTPN_REQUIRE(fx > 0 && fy > 0, "%s: image %d: scale (%g, %g) must be > 0", fn, b, fx, fy);
  CTPN_REQUIRE(sh * fy < 1e9 && sw * fx < 1e9, "%s: image %d: scale (%g, %g) too large", fn, b, fx, fy);
  if (ctpn_resize_out_size(sh, sw, fx, fy, eh, ew)) {
    set_error("%s: image %d: %d x %d at (%g, %g) resizes to nothing", fn, b, sh, sw, fx, fy);
    return CTPN_ERR_INVALID;
  }
  CTPN_REQUIRE(*eh == dst_hw[2 * b] && *ew == dst_hw[2 * b + 1], "%s: image %d: dst is %d x %d, cv2 would produce %d x %d", fn,
               b, dst_hw[2 * b], dst_hw[2 * b + 1], *eh, *ew);
  CTPN_REQUIRE(*eh <= H && *ew <= W, "%s: image %d: output %d x %d does not fit the %d x %d canvas", fn, b, *eh, *ew, H, W);
  return CTPN_OK;
}

// Validates the per-image host descriptors of a ragged call and fills the kernel's parameter struct; no CUDA call.
// stored (NULL: every row): how many of image b's rows the source holds (row-compacted sources).
static int ragged_params(const char *fn, size_t src_elems, const long long *src_offset, const int *src_hwp, const double *fxy,
                         const int *dst_hw, int B, int C, int H, int W, RaggedResize *p, long long *max_pixels,
                         const int *stored = nullptr) {
  CTPN_REQUIRE(src_offset && src_hwp && fxy && dst_hw, "%s: null descriptor array", fn);
  CTPN_REQUIRE(B >= 1 && B <= kRaggedMax, "%s: B = %d, must be 1..%d", fn, B, kRaggedMax);
  CTPN_REQUIRE(H > 0 && W > 0, "%s: bad canvas %d x %d", fn, H, W);
  memset(p, 0, sizeof(*p));
  p->H = H;
  p->W = W;
  p->C = C;
  *max_pixels = 0;
  for (int b = 0; b < B; ++b) {
    const int sh = src_hwp[3 * b], sw = src_hwp[3 * b + 1], pitch = src_hwp[3 * b + 2];
    const double fx = fxy[2 * b], fy = fxy[2 * b + 1];
    const long long off = src_offset[b];
    CTPN_REQUIRE(sh > 0 && sw > 0, "%s: image %d: bad source size %d x %d", fn, b, sh, sw);
    CTPN_REQUIRE(pitch >= sw, "%s: image %d: row pitch %d < width %d", fn, b, pitch, sw);
    CTPN_REQUIRE(off >= 0, "%s: image %d: negative source offset %lld", fn, b, off);
    const int held = stored ? stored[b] : sh;
    CTPN_REQUIRE(held >= 1 && held <= sh, "%s: image %d: %d stored rows, must be 1..%d (the source height)", fn, b, held, sh);
    const unsigned __int128 end = (unsigned __int128)off +
                                  ((unsigned __int128)(held - 1) * (unsigned)pitch + (unsigned)sw) * (unsigned)C;
    CTPN_REQUIRE(end <= (unsigned __int128)src_elems, "%s: image %d: source extent ends at %llu, past src_elems = %zu", fn, b,
                 (unsigned long long)end, src_elems);
    int eh = 0, ew = 0;
    const int rc = ragged_geometry_ok(fn, b, sh, sw, fx, fy, dst_hw, H, W, &eh, &ew);
    if (rc) return rc;
    p->src_offset[b] = off;
    p->sh[b] = sh;
    p->sw[b] = sw;
    p->pitch[b] = pitch;
    p->dh[b] = eh;
    p->dw[b] = ew;
    p->scale_x[b] = 1.0 / fx;
    p->scale_y[b] = 1.0 / fy;
    if (p->scale_x[b] == 2.0 && p->scale_y[b] == 2.0) p->area2 |= 1ull << b;   // as the single-image entry points route it
    *max_pixels = std::max(*max_pixels, (long long)eh * ew);
  }
  return CTPN_OK;
}

// grid (x, B): about 32 CTAs per SM over the whole batch, no more x-blocks than the largest image needs
static int ragged_grid(int B, long long max_pixels, dim3 *grid) {
  int sms = 0, rc;
  if ((rc = current_sm_count(&sms))) return rc;
  const long long per_image = std::max(1LL, 32LL * sms / B);
  *grid = dim3((unsigned)std::min<long long>((max_pixels + 255) / 256, per_image), (unsigned)B);
  return CTPN_OK;
}

extern "C" int ctpn_resize_linear_u8_ragged(const void *src, size_t src_elems, const long long *src_offset, const int *src_hwp,
                                            const double *fxy, const int *dst_hw, int B, int channels, void *dst, int H, int W,
                                            void *stream) {
  CTPN_REQUIRE(src && dst, "ctpn_resize_linear_u8_ragged: null pointer");
  CTPN_REQUIRE(channels > 0 && channels <= 4, "ctpn_resize_linear_u8_ragged: bad channel count %d", channels);
  RaggedResize p;
  long long max_pixels = 0, work = 0;
  int rc = ragged_params("ctpn_resize_linear_u8_ragged", src_elems, src_offset, src_hwp, fxy, dst_hw, B, channels, H, W, &p,
                         &max_pixels);
  if (rc) return rc;
  dim3 grid;
  if ((rc = ragged_grid(B, max_pixels, &grid))) return rc;
  for (int b = 0; b < B; ++b) work += (long long)p.dh[b] * p.dw[b] * channels;
  ProfScope prof("resize_linear_u8_ragged", (double)work, (cudaStream_t)stream);
  resize_linear_u8_ragged_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint8_t *)src, (uint8_t *)dst, p);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

extern "C" int ctpn_resize_linear_u8_ragged_rows(const void *src, size_t src_elems, const long long *src_offset, const int *src_hwp,
                                                 const int *stored_rows, const int *row_map, size_t map_elems,
                                                 const long long *map_offset, const double *fxy, const int *dst_hw, int B,
                                                 int channels, void *dst, int H, int W, void *stream) {
  const char *fn = "ctpn_resize_linear_u8_ragged_rows";
  CTPN_REQUIRE(src && dst && row_map, "%s: null pointer", fn);
  CTPN_REQUIRE(stored_rows && map_offset, "%s: null descriptor array", fn);
  CTPN_REQUIRE(channels > 0 && channels <= 4, "%s: bad channel count %d", fn, channels);
  RaggedResizeRows q;
  long long max_pixels = 0, work = 0;
  int rc = ragged_params(fn, src_elems, src_offset, src_hwp, fxy, dst_hw, B, channels, H, W, &q.r, &max_pixels, stored_rows);
  if (rc) return rc;
  memset(q.map_offset, 0, sizeof(q.map_offset));
  memset(q.stored, 0, sizeof(q.stored));
  for (int b = 0; b < B; ++b) {
    const long long off = map_offset[b];
    CTPN_REQUIRE(off >= 0 && (unsigned long long)off <= map_elems && (size_t)q.r.sh[b] <= map_elems - (size_t)off,
                 "%s: image %d: row map [%lld, %lld + %d) lies outside map_elems = %zu", fn, b, off, off, q.r.sh[b], map_elems);
    q.map_offset[b] = off;
    q.stored[b] = stored_rows[b];
  }
  dim3 grid;
  if ((rc = ragged_grid(B, max_pixels, &grid))) return rc;
  for (int b = 0; b < B; ++b) work += (long long)q.r.dh[b] * q.r.dw[b] * channels;
  ProfScope prof("resize_linear_u8_ragged_rows", (double)work, (cudaStream_t)stream);
  resize_linear_u8_ragged_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint8_t *)src, row_map, (uint8_t *)dst, q);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

extern "C" int ctpn_image_blob_f32_ragged(const void *src_u8, size_t src_elems, const long long *src_offset, const int *src_hwp,
                                          const double *fxy, const int *dst_hw, const float *lut, int B, float *dst, int H, int W,
                                          void *stream) {
  CTPN_REQUIRE(src_u8 && lut && dst, "ctpn_image_blob_f32_ragged: null pointer");
  RaggedResize p;
  long long max_pixels = 0, work = 0;
  int rc = ragged_params("ctpn_image_blob_f32_ragged", src_elems, src_offset, src_hwp, fxy, dst_hw, B, 3, H, W, &p, &max_pixels);
  if (rc) return rc;
  dim3 grid;
  if ((rc = ragged_grid(B, max_pixels, &grid))) return rc;
  for (int b = 0; b < B; ++b) work += (long long)p.dh[b] * p.dw[b] * 3;
  ProfScope prof("image_blob_f32_ragged", (double)work, (cudaStream_t)stream);
  image_blob_f32_ragged_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint8_t *)src_u8, lut, dst, p);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

extern "C" int ctpn_resize_linear_u8_strided(const void *const *src, const size_t *src_bytes, const long long *src_offset,
                                             const long long *src_strides, const int *src_hw, const double *fxy,
                                             const int *dst_hw, int B, void *dst, int H, int W, void *stream) {
  const char *fn = "ctpn_resize_linear_u8_strided";
  CTPN_REQUIRE(dst, "%s: null pointer", fn);
  CTPN_REQUIRE(src && src_bytes && src_offset && src_strides && src_hw && fxy && dst_hw, "%s: null descriptor array", fn);
  CTPN_REQUIRE(B >= 1 && B <= kRaggedMax, "%s: B = %d, must be 1..%d", fn, B, kRaggedMax);
  CTPN_REQUIRE(H > 0 && W > 0, "%s: bad canvas %d x %d", fn, H, W);
  StridedResize p;
  memset(&p, 0, sizeof(p));
  p.H = H;
  p.W = W;
  long long max_pixels = 0, work = 0;
  for (int b = 0; b < B; ++b) {
    const int sh = src_hw[2 * b], sw = src_hw[2 * b + 1];
    StridedPixels px;
    int rc = strided_source(fn, b, src[b], src_bytes[b], src_offset[b], src_strides + 3 * b, sh, sw, &px);
    if (rc) return rc;
    int eh = 0, ew = 0;
    if ((rc = ragged_geometry_ok(fn, b, sh, sw, fxy[2 * b], fxy[2 * b + 1], dst_hw, H, W, &eh, &ew))) return rc;
    p.base[b] = px.base;
    p.row_stride[b] = px.row_stride;
    p.col_stride[b] = px.col_stride;
    p.chan_stride[b] = px.chan_stride;
    p.sh[b] = sh;
    p.sw[b] = sw;
    p.dh[b] = eh;
    p.dw[b] = ew;
    p.scale_x[b] = 1.0 / fxy[2 * b];
    p.scale_y[b] = 1.0 / fxy[2 * b + 1];
    if (p.scale_x[b] == 2.0 && p.scale_y[b] == 2.0) p.area2 |= 1ull << b;
    max_pixels = std::max(max_pixels, (long long)eh * ew);
    work += (long long)eh * ew * 3;
  }
  dim3 grid;
  int rc = ragged_grid(B, max_pixels, &grid);
  if (rc) return rc;
  ProfScope prof("resize_linear_u8_strided", (double)work, (cudaStream_t)stream);
  resize_linear_u8_strided_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((uint8_t *)dst, p);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

extern "C" int ctpn_resize_linear_u8_yuv420(const void *const *planes, const size_t *plane_bytes, const long long *plane_offset,
                                            const long long *plane_strides, const int *src_hw, const double *fxy,
                                            const int *dst_hw, int B, void *dst, int H, int W, void *stream) {
  const char *fn = "ctpn_resize_linear_u8_yuv420";
  CTPN_REQUIRE(dst, "%s: null pointer", fn);
  CTPN_REQUIRE(planes && plane_bytes && plane_offset && plane_strides && src_hw && fxy && dst_hw, "%s: null descriptor array",
               fn);
  CTPN_REQUIRE(B >= 1 && B <= kRaggedMax, "%s: B = %d, must be 1..%d", fn, B, kRaggedMax);
  CTPN_REQUIRE(H > 0 && W > 0, "%s: bad canvas %d x %d", fn, H, W);
  Yuv420Resize chunk[(kRaggedMax + kYuvChunk - 1) / kYuvChunk];
  memset(chunk, 0, sizeof(chunk));
  long long max_pixels[(kRaggedMax + kYuvChunk - 1) / kYuvChunk] = {}, work = 0;
  for (int b = 0; b < B; ++b) {
    const int sh = src_hw[2 * b], sw = src_hw[2 * b + 1];
    Yuv420Pixels px;
    int rc = yuv420_source(fn, b, planes + 3 * b, plane_bytes + 3 * b, plane_offset + 3 * b, plane_strides + 6 * b, sh, sw, &px);
    if (rc) return rc;
    Yuv420Resize &p = chunk[b / kYuvChunk];
    const int k = b % kYuvChunk;
    const uint8_t *const pl[3] = {px.y, px.u, px.v};
    const long long rs[3] = {px.y_row, px.u_row, px.v_row};
    const int cs[3] = {px.y_col, px.u_col, px.v_col};
    for (int q = 0; q < 3; ++q) {
      p.plane[k][q] = pl[q];
      p.row_stride[k][q] = rs[q];
      p.col_stride[k][q] = cs[q];
    }
    int eh = 0, ew = 0;
    if ((rc = ragged_geometry_ok(fn, b, sh, sw, fxy[2 * b], fxy[2 * b + 1], dst_hw, H, W, &eh, &ew))) return rc;
    p.H = H;
    p.W = W;
    p.sh[k] = sh;
    p.sw[k] = sw;
    p.dh[k] = eh;
    p.dw[k] = ew;
    p.scale_x[k] = 1.0 / fxy[2 * b];
    p.scale_y[k] = 1.0 / fxy[2 * b + 1];
    if (p.scale_x[k] == 2.0 && p.scale_y[k] == 2.0) p.area2 |= 1u << k;
    max_pixels[b / kYuvChunk] = std::max(max_pixels[b / kYuvChunk], (long long)eh * ew);
    work += (long long)eh * ew * 3;
  }
  ProfScope prof("resize_linear_u8_yuv420", (double)work, (cudaStream_t)stream);
  for (int first = 0; first < B; first += kYuvChunk) {
    const int nb = std::min(kYuvChunk, B - first);
    dim3 grid;
    int rc = ragged_grid(nb, max_pixels[first / kYuvChunk], &grid);
    if (rc) return rc;
    resize_linear_u8_yuv420_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((uint8_t *)dst + (size_t)first * H * W * 3,
                                                                            chunk[first / kYuvChunk]);
    CTPN_LAUNCH_CHECK();
  }
  return CTPN_OK;
}
