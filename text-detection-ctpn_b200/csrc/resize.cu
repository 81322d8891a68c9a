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
// sources that hold only the rows it reads (Engine.stream_rois_images uploads camera photos that way).
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

// Where source row y of an image is stored: every row in place ...
struct DenseRows {
  __device__ __forceinline__ int operator()(int y) const { return y; }
};
// ... or only the rows the resize reads (ctpn_resize_linear_u8_ragged_rows): map[y] is the stored index of source row y.
// The map is device memory the host never saw, so the index is clamped to the stored extent the host did check.
struct CompactRows {
  const int *__restrict__ map;
  int stored;
  __device__ __forceinline__ int operator()(int y) const { return min(max(__ldg(map + y), 0), stored - 1); }
};

// One output pixel of cv2.resize(INTER_LINEAR) of a uint8 image im [sh][pitch][C] (pitch >= sw pixels per row) -> o[C].
// Shared by the uniform and the ragged kernels: the ragged batch is bit-identical to single-image runs by construction.
// Taps, weights and border clamping come from the source geometry (sh, sw); only the address of a row goes through
// `row`.
template <class Rows>
__device__ __forceinline__ void resize_u8_pixel(const uint8_t *__restrict__ im, int sh, int sw, int pitch, int C, int dx, int dy,
                                                double scale_x, double scale_y, bool area2, uint8_t *__restrict__ o,
                                                const Rows row) {
  if (area2) {
    const int y0 = 2 * dy, x0 = 2 * dx;
    const int ny = min(2, sh - y0), nx = min(2, sw - x0);
    for (int c = 0; c < C; ++c) {
      int sum = 0;
      for (int yy = 0; yy < ny; ++yy)
        for (int xx = 0; xx < nx; ++xx) sum += im[((size_t)row(y0 + yy) * pitch + x0 + xx) * C + c];
      int v = (ny * nx == 4) ? (sum + 2) >> 2 : __float2int_rn(__fdiv_rn((float)sum, (float)(ny * nx)));
      o[c] = (uint8_t)min(max(v, 0), 255);
    }
    return;
  }
  int sx0, sx1, a0, a1, sy0, sy1, b0, b1;
  resize_taps(dx, sw, scale_x, true, sx0, sx1, a0, a1);
  resize_taps(dy, sh, scale_y, false, sy0, sy1, b0, b1);
  const uint8_t *r0 = im + (size_t)row(sy0) * pitch * C, *r1 = im + (size_t)row(sy1) * pitch * C;
  for (int c = 0; c < C; ++c) {
    const int h0 = r0[(size_t)sx0 * C + c] * a0 + r0[(size_t)sx1 * C + c] * a1;
    const int h1 = r1[(size_t)sx0 * C + c] * a0 + r1[(size_t)sx1 * C + c] * a1;
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
    resize_u8_pixel(src + (size_t)b * sh * sw * C, sh, sw, sw, C, dx, dy, scale_x, scale_y, area2 != 0, dst + (size_t)i * C,
                    DenseRows());
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
    resize_u8_pixel(im, p.sh[b], p.sw[b], p.pitch[b], C, dx, dy, p.scale_x[b], p.scale_y[b], (p.area2 >> b) & 1,
                    out + ((size_t)dy * p.W + dx) * C, DenseRows());
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
  const CompactRows row{rows + q.map_offset[b], q.stored[b]};
  uint8_t *out = dst + (size_t)b * p.H * p.W * C;
  const long long total = (long long)dh * dw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int dx = (int)(i % dw), dy = (int)(i / dw);
    resize_u8_pixel(im, p.sh[b], p.sw[b], p.pitch[b], C, dx, dy, p.scale_x[b], p.scale_y[b], (p.area2 >> b) & 1,
                    out + ((size_t)dy * p.W + dx) * C, row);
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
    CTPN_REQUIRE(fx > 0 && fy > 0, "%s: image %d: scale (%g, %g) must be > 0", fn, b, fx, fy);
    CTPN_REQUIRE(sh * fy < 1e9 && sw * fx < 1e9, "%s: image %d: scale (%g, %g) too large", fn, b, fx, fy);
    CTPN_REQUIRE(off >= 0, "%s: image %d: negative source offset %lld", fn, b, off);
    const int held = stored ? stored[b] : sh;
    CTPN_REQUIRE(held >= 1 && held <= sh, "%s: image %d: %d stored rows, must be 1..%d (the source height)", fn, b, held, sh);
    const unsigned __int128 end = (unsigned __int128)off +
                                  ((unsigned __int128)(held - 1) * (unsigned)pitch + (unsigned)sw) * (unsigned)C;
    CTPN_REQUIRE(end <= (unsigned __int128)src_elems, "%s: image %d: source extent ends at %llu, past src_elems = %zu", fn, b,
                 (unsigned long long)end, src_elems);
    int eh = 0, ew = 0;
    if (ctpn_resize_out_size(sh, sw, fx, fy, &eh, &ew)) {
      set_error("%s: image %d: %d x %d at (%g, %g) resizes to nothing", fn, b, sh, sw, fx, fy);
      return CTPN_ERR_INVALID;
    }
    CTPN_REQUIRE(eh == dst_hw[2 * b] && ew == dst_hw[2 * b + 1], "%s: image %d: dst is %d x %d, cv2 would produce %d x %d", fn, b,
                 dst_hw[2 * b], dst_hw[2 * b + 1], eh, ew);
    CTPN_REQUIRE(eh <= H && ew <= W, "%s: image %d: output %d x %d does not fit the %d x %d canvas", fn, b, eh, ew, H, W);
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
