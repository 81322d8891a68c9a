// ctpn_net_*: the CTPN test graph up to the two head tensors, as one stream-ordered sequence of
// the stage kernels (lib/networks/VGGnet_test.py:16-52; variable names per SURVEY.md App. A.2).
//   uint8 image -> conv1_1 (wgmma, fused mean subtraction) -> 13 x wgmma conv (+fused pools)
//   -> x-projection GEMM -> BiLSTM recurrence (2-CTA clusters) -> FC GEMM -> heads GEMM.
// Weights live in library-owned device memory; activations in the caller's workspace.
#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include <cuda_fp8.h>

#include <cmath>

#include "common.cuh"
#ifdef CTPN_DEBUG
#include "testing/ctpn_b200_testing.h"
#endif

namespace ctpn {

struct ConvSpec { const char *name; int cin, cout; bool pool; };
static const ConvSpec kConvs[14] = {
    {"conv1_1", 3, 64, false},    {"conv1_2", 64, 64, true},    {"conv2_1", 64, 128, false},
    {"conv2_2", 128, 128, true},  {"conv3_1", 128, 256, false}, {"conv3_2", 256, 256, false},
    {"conv3_3", 256, 256, true},  {"conv4_1", 256, 512, false}, {"conv4_2", 512, 512, false},
    {"conv4_3", 512, 512, true},  {"conv5_1", 512, 512, false}, {"conv5_2", 512, 512, false},
    {"conv5_3", 512, 512, false}, {"rpn_conv/3x3", 512, 512, false}};
static const char *kFw = "lstm_o/bidirectional_rnn/fw/lstm_cell";
static const char *kBw = "lstm_o/bidirectional_rnn/bw/lstm_cell";
static const double kPixelMeans[3] = {102.9801, 115.9465, 122.7717};   // lib/fast_rcnn/config.py:200 (BGR)

struct Tap { const void *ptr; long long pixels; int channels; bool planes; float q_s = 0.f, q_t = 0.f; int stack_h = 0, stack_w = 0; };   // q_s > 0: F16F8 planes; stack_h > 0: rows stacked as [B][h + 1][w]

}  // namespace ctpn

using namespace ctpn;

struct ctpn_net {
  int planes = 2;
  // F16F8 arithmetic for the 3x3 layers (planes = CTPN_ARITH_F16F8 at creation; common.cuh).  The matmuls around the
  // BiLSTM (0.9 % of the FLOPs) stay on two bf16 planes.  Per-layer power-of-two scales: w_s / w_t from max|w| at
  // finalize time; act_s / act_t (quantisation of the layer's OUTPUT) from the first batch seen (calibrate()).
  bool f16f8 = false, calibrated = false;
  bool promote = false;     // CTPN_ARITH_BF16X3P: planes = 3 with CTPN_F_PROMOTE on every conv_tc layer
  float w_s[14] = {0}, w_t[14] = {0}, act_s[14] = {0}, act_t[14] = {0}, act_max[14] = {0};
  unsigned *absmax_dev = nullptr;
  int conv_simt = 0, conv1_simt = 0, keep = 0;
  std::map<std::string, std::vector<float>> host;
  bool dirty = true;
  std::vector<void *> owned;
  float *c11_w = nullptr, *c11_b = nullptr, *lut = nullptr;
  void *conv_w[14] = {nullptr};
  float *conv_b[14] = {nullptr};
  void *xproj_w = nullptr, *fc_w = nullptr, *head_w = nullptr;
  float *xproj_b = nullptr, *fc_b = nullptr, *head_b = nullptr, *wh_fw = nullptr, *wh_bw = nullptr;
  std::map<std::string, Tap> taps;
};

namespace ctpn {

static int dev_alloc(ctpn_net *n, void **p, size_t bytes) {
  CTPN_CUDA(cudaMalloc(p, bytes));
  n->owned.push_back(*p);
  return CTPN_OK;
}

static int upload(ctpn_net *n, float **dst, const float *src, size_t count) {
  int rc = dev_alloc(n, (void **)dst, count * sizeof(float));
  if (rc) return rc;
  CTPN_CUDA(cudaMemcpy(*dst, src, count * sizeof(float), cudaMemcpyHostToDevice));
  return CTPN_OK;
}

// upload a TF-layout [taps][cin][cout] float32 matrix and convert it to bf16 planes
static int upload_packed(ctpn_net *n, void **dst, const float *src, int taps, int cin, int cout, int cout_pad) {
  float *tmp = nullptr;
  const size_t cnt = (size_t)taps * cin * cout;
  CTPN_CUDA(cudaMalloc(&tmp, cnt * sizeof(float)));
  cudaError_t e = cudaMemcpy(tmp, src, cnt * sizeof(float), cudaMemcpyHostToDevice);
  int rc = e == cudaSuccess ? dev_alloc(n, dst, (size_t)n->planes * cout_pad * taps * cin * 2) : cuda_fail(e, "memcpy", __FILE__, __LINE__);
  if (!rc) rc = ctpn_pack_weights(tmp, taps, cin, cout, cout_pad, n->planes, *dst, nullptr);
  if (!rc) { e = cudaDeviceSynchronize(); if (e != cudaSuccess) rc = cuda_fail(e, "sync", __FILE__, __LINE__); }
  cudaFree(tmp);
  return rc;
}

// upload a TF-layout [9][cin][cout] float32 kernel in the F16F8 weight format with scales from max|w|
static int upload_packed_f16f8(ctpn_net *n, void **dst, const float *src, int cin, int cout, float *s_w, float *t_w) {
  const size_t cnt = (size_t)9 * cin * cout;
  float mx = 0.f;
  for (size_t i = 0; i < cnt; ++i) mx = std::max(mx, fabsf(src[i]));
  if (!(mx > 0.f) || !std::isfinite(mx)) { set_error("weights are all zero or not finite"); return CTPN_ERR_INVALID; }
  *s_w = exp2f(floorf(log2f(16384.f / mx)));      // fp16(w s_w) stays below 2^15
  *t_w = exp2f(floorf(log2f(448.f / mx)));        // e4m3(w t_w) uses the top binade
  float *tmp = nullptr;
  CTPN_CUDA(cudaMalloc(&tmp, cnt * sizeof(float)));
  cudaError_t e = cudaMemcpy(tmp, src, cnt * sizeof(float), cudaMemcpyHostToDevice);
  int rc = e == cudaSuccess ? dev_alloc(n, dst, (size_t)2 * cout * 9 * cin * 2) : cuda_fail(e, "memcpy", __FILE__, __LINE__);
  if (!rc) rc = ctpn_pack_weights_f16f8(tmp, 9, cin, cout, cout, *s_w, *t_w, *dst, nullptr);
  if (!rc) { e = cudaDeviceSynchronize(); if (e != cudaSuccess) rc = cuda_fail(e, "sync", __FILE__, __LINE__); }
  cudaFree(tmp);
  return rc;
}

static void free_device(ctpn_net *n) {
  for (void *p : n->owned) cudaFree(p);
  n->owned.clear();
  n->absmax_dev = nullptr;
  n->calibrated = false;
}

static const std::vector<float> *need(ctpn_net *n, const std::string &name, size_t count) {
  auto it = n->host.find(name);
  if (it == n->host.end()) { set_error("weight '%s' has not been set", name.c_str()); return nullptr; }
  if (it->second.size() != count) {
    set_error("weight '%s' has %zu elements, expected %zu", name.c_str(), it->second.size(), count);
    return nullptr;
  }
  return &it->second;
}

static int finalize(ctpn_net *n) {
  if (!n->dirty) return CTPN_OK;
  free_device(n);
  int rc;
  // mean-subtraction table: float32(double(v) - mean), numpy's in-place `im -= PIXEL_MEANS` (test.py:9)
  {
    std::vector<float> lut(256 * 3);
    for (int v = 0; v < 256; ++v)
      for (int c = 0; c < 3; ++c) lut[v * 3 + c] = (float)((double)v - kPixelMeans[c]);
    if ((rc = upload(n, &n->lut, lut.data(), lut.size()))) return rc;
  }
  for (int l = 0; l < 14; ++l) {
    const ConvSpec &s = kConvs[l];
    const auto *w = need(n, std::string(s.name) + "/weights", (size_t)9 * s.cin * s.cout);
    const auto *b = need(n, std::string(s.name) + "/biases", s.cout);
    if (!w || !b) return CTPN_ERR_INVALID;
    if (l == 0) {
      if ((rc = upload(n, &n->c11_w, w->data(), w->size()))) return rc;
      if ((rc = upload(n, &n->c11_b, b->data(), b->size()))) return rc;
    } else {
      if (n->f16f8) rc = upload_packed_f16f8(n, &n->conv_w[l], w->data(), s.cin, s.cout, &n->w_s[l], &n->w_t[l]);
      else rc = upload_packed(n, &n->conv_w[l], w->data(), 9, s.cin, s.cout, s.cout);
      if (rc) return rc;
      if ((rc = upload(n, &n->conv_b[l], b->data(), b->size()))) return rc;
    }
  }
  {   // LSTM: kernel rows 0..511 multiply x (-> x-projection GEMM), rows 512..639 multiply h
    const auto *kf = need(n, std::string(kFw) + "/kernel", 640 * 512), *kb = need(n, std::string(kBw) + "/kernel", 640 * 512);
    const auto *bf = need(n, std::string(kFw) + "/bias", 512), *bb = need(n, std::string(kBw) + "/bias", 512);
    if (!kf || !kb || !bf || !bb) return CTPN_ERR_INVALID;
    std::vector<float> wx((size_t)512 * 1024), bx(1024);
    for (int k = 0; k < 512; ++k)
      for (int c = 0; c < 512; ++c) {
        wx[(size_t)k * 1024 + c] = (*kf)[(size_t)k * 512 + c];
        wx[(size_t)k * 1024 + 512 + c] = (*kb)[(size_t)k * 512 + c];
      }
    for (int c = 0; c < 512; ++c) { bx[c] = (*bf)[c]; bx[512 + c] = (*bb)[c]; }
    if ((rc = upload_packed(n, &n->xproj_w, wx.data(), 1, 512, 1024, 1024))) return rc;
    if ((rc = upload(n, &n->xproj_b, bx.data(), bx.size()))) return rc;
    if ((rc = upload(n, &n->wh_fw, kf->data() + 512 * 512, 128 * 512))) return rc;
    if ((rc = upload(n, &n->wh_bw, kb->data() + 512 * 512, 128 * 512))) return rc;
  }
  {
    const auto *w = need(n, "lstm_o/weights", 256 * 512), *b = need(n, "lstm_o/biases", 512);
    if (!w || !b) return CTPN_ERR_INVALID;
    if ((rc = upload_packed(n, &n->fc_w, w->data(), 1, 256, 512, 512))) return rc;
    if ((rc = upload(n, &n->fc_b, b->data(), b->size()))) return rc;
  }
  {   // heads share one GEMM: columns 0..39 rpn_bbox_pred, 40..59 rpn_cls_score, 60..63 zero padding
    const auto *wb = need(n, "rpn_bbox_pred/weights", 512 * 40), *bb = need(n, "rpn_bbox_pred/biases", 40);
    const auto *wc = need(n, "rpn_cls_score/weights", 512 * 20), *bc = need(n, "rpn_cls_score/biases", 20);
    if (!wb || !bb || !wc || !bc) return CTPN_ERR_INVALID;
    std::vector<float> w((size_t)512 * 64, 0.f), b(64, 0.f);
    for (int k = 0; k < 512; ++k) {
      for (int c = 0; c < 40; ++c) w[(size_t)k * 64 + c] = (*wb)[(size_t)k * 40 + c];
      for (int c = 0; c < 20; ++c) w[(size_t)k * 64 + 40 + c] = (*wc)[(size_t)k * 20 + c];
    }
    for (int c = 0; c < 40; ++c) b[c] = (*bb)[c];
    for (int c = 0; c < 20; ++c) b[40 + c] = (*bc)[c];
    if ((rc = upload_packed(n, &n->head_w, w.data(), 1, 512, 64, 64))) return rc;
    if ((rc = upload(n, &n->head_b, b.data(), b.size()))) return rc;
  }
  if (n->f16f8 && (rc = dev_alloc(n, (void **)&n->absmax_dev, sizeof(unsigned)))) return rc;
  n->dirty = false;
  return CTPN_OK;
}

struct NetLayout {
  bool stack;           // conv4_3's pooled output and conv5_1..conv5_3 outputs are row-stacked ([B][h + 1][w], zero pad rows)
  size_t act[16];       // offsets of the 14 conv outputs + lstm_out + fc_out
  size_t xproj, heads, total;
  int h[15], w[15];     // spatial size of each conv output
  int fh, fw;
};

static NetLayout net_layout(const ctpn_net *n, int B, int H, int W) {
  NetLayout L;
  const int P = n->planes;
  size_t sizes[16];
  int h = H, w = W;
  for (int l = 0; l < 14; ++l) {
    if (kConvs[l].pool) { h /= 2; w /= 2; }
    L.h[l] = h; L.w[l] = w;
    sizes[l] = (size_t)P * B * h * w * kConvs[l].cout * 2;
  }
  L.fh = h; L.fw = w;
  // stack the 1/16-scale maps when one tall image needs fewer 16-row tiles than B separate ones (37 rows: 76 vs 96 at B = 32)
  L.stack = !n->conv_simt && ((long long)B * (h + 1) + 15) / 16 < (long long)B * ((h + 15) / 16);   // (the SIMT reference kernels of the test library know no stacking)
  if (L.stack)
    for (int l = 9; l <= 12; ++l) sizes[l] = (size_t)P * B * (h + 1) * w * kConvs[l].cout * 2;
  const size_t M = (size_t)B * h * w;
  sizes[14] = (size_t)P * M * 256 * 2;   // lstm_out
  sizes[15] = (size_t)P * M * 512 * 2;   // lstm_o (FC)
  size_t o = 0;
  if (n->keep) {
    for (int i = 0; i < 16; ++i) { L.act[i] = o; o = align_up(o + sizes[i], 1024); }
  } else {   // ping-pong between two buffers
    size_t even = 0, odd = 0;
    for (int i = 0; i < 16; ++i) (i & 1 ? odd : even) = std::max(i & 1 ? odd : even, sizes[i]);
    even = align_up(even, 1024); odd = align_up(odd, 1024);
    for (int i = 0; i < 16; ++i) L.act[i] = (i & 1) ? even : 0;
    o = even + odd;
  }
  L.xproj = o; o = align_up(o + M * 1024 * sizeof(float), 1024);
  L.heads = o; o = align_up(o + M * 64 * sizeof(float), 1024);
  L.total = o;
  return L;
}

__global__ void split_heads_kernel(const float *__restrict__ heads, long long M, float *__restrict__ cls, float *__restrict__ bbox) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * 64) return;
  const long long m = i >> 6;
  const int c = (int)(i & 63);
  const float v = heads[i];
  if (c < 40) bbox[m * 40 + c] = v;
  else if (c < 60) cls[m * 20 + (c - 40)] = v;
}

// F16F8 planes -> float32: (h + residual / (2^11 t / s)) / s
__global__ void f16f8_to_f32_kernel(const __half *__restrict__ hi, const uint8_t *__restrict__ cross, long long n, int C, float s, float t,
                                    int stack_h, int stack_w, float *__restrict__ dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  long long pix = i / C;
  const int c = (int)(i % C);
  if (stack_h) {     // compact pixel index -> position in the stacked frame [B][stack_h + 1][stack_w]
    const long long per = (long long)stack_h * stack_w, b = pix / per, r = pix % per;
    pix = b * (stack_h + 1) * stack_w + r;
  }
  const uint8_t rb = cross[pix * 2 * C + (c >> 6) * 128 + 64 + (c & 63)];
  const __half_raw hr = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)rb, __NV_E4M3);
  const float r = __half2float(__half(hr)) / (kResidualGain * t / s);
  dst[i] = (__half2float(hi[pix * C + c]) + r) / s;
}

__global__ void planes_to_f32_kernel(const __nv_bfloat16 *__restrict__ src, long long n, long long plane_stride, int planes, int C,
                                     int stack_h, int stack_w, float *__restrict__ dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  long long j = i;
  if (stack_h) {     // compact element index -> position in the stacked frame [B][stack_h + 1][stack_w][C]
    const long long pix = i / C, per = (long long)stack_h * stack_w;
    j = ((pix / per) * (stack_h + 1) * stack_w + pix % per) * C + i % C;
  }
  float v = __bfloat162float(src[j]);
  if (planes > 1) v += __bfloat162float(src[j + plane_stride]);
  if (planes > 2) v += __bfloat162float(src[j + 2 * plane_stride]);
  dst[i] = v;
}

// max |x| over an fp16 tensor (non-negative floats order like their bit patterns; Inf / NaN come out on top)
__global__ void absmax_f16_kernel(const __half *__restrict__ x, long long n, unsigned *__restrict__ out) {
  float m = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(__half2float(x[i])));
  unsigned bits = __float_as_uint(m);
  if (m != m) bits = 0x7fc00000u;
  for (int o = 16; o; o >>= 1) bits = max(bits, __shfl_xor_sync(0xffffffffu, bits, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, bits);
}

// pools before the output of layer l: a ragged batch's image of size (h, w) covers (h >> k, w >> k) of that output
static int out_level(int l) {
  int k = 0;
  for (int i = 0; i <= l; ++i) k += kConvs[i].pool ? 1 : 0;
  return k;
}

// one 3x3 layer in the F16F8 arithmetic with the scales currently in the net (sizes: ragged batch, or null)
static int run_layer_f16f8(ctpn_net *n, int l, const void *in, void *out, int B, int h, int w, bool stack, const int *sizes, void *stream) {
  const ConvSpec &s = kConvs[l];
  int flags = CTPN_F_RELU | (s.pool ? CTPN_F_POOL : 0) | (l == 13 ? CTPN_F_OUT_BF16X2 : 0);   // rpn_conv feeds the bf16x2 matmuls
  if (stack && l >= 9 && l <= 12) flags |= CTPN_F_STACK_OUT;
  if (stack && l >= 10) flags |= CTPN_F_STACK_IN;
  const float inv_main = 1.f / (n->act_s[l - 1] * n->w_s[l]), inv_cross = 1.f / (kResidualGain * n->act_t[l - 1] * n->w_t[l]);
  return conv3x3_f16f8_ragged(in, n->conv_w[l], n->conv_b[l], out, B, h, w, s.cin, s.cout, 9, flags, inv_main, inv_cross,
                              l == 13 ? 1.f : n->act_s[l], l == 13 ? 1.f : n->act_t[l], sizes, out_level(l), stream);
}

// Activation scales from data: every layer is run with provisional scales, the maximum of its fp16 plane is read back,
// the scales are fixed (fp16 plane below 2^14, e4m3 copy two binades below saturation) and the layer is run again so the
// next one sees its final input.  Synchronises per layer; happens once (first forward, or after "recalibrate").
static int calibrate_f16f8(ctpn_net *n, const void *images, int src_is_f32, const int *sizes, int B, int H, int W, const NetLayout &L,
                           char *ws, void *stream) {
  cudaStream_t st = (cudaStream_t)stream;
  int h = H, w = W;
  for (int l = 0; l < 13; ++l) {
    const void *in = l == 0 ? images : (const void *)(ws + L.act[l - 1]);
    if (L.stack && l == 9)      // pad rows of conv4_3's stacked output (see ctpn_net_forward)
      CTPN_CUDA(cudaMemsetAsync(ws + L.act[9], 0, (size_t)n->planes * B * (L.h[9] + 1) * L.w[9] * kConvs[9].cout * 2, st));
    float s_try = 1.f;
    for (int attempt = 0; ; ++attempt) {
      n->act_s[l] = s_try; n->act_t[l] = 1.f;
      int rc = l == 0 ? conv1_1_tc_ragged(images, src_is_f32, n->lut, n->c11_w, n->c11_b, ws + L.act[0], B, h, w, 2, true, s_try, 1.f, sizes, stream)
                      : run_layer_f16f8(n, l, in, ws + L.act[l], B, h, w, L.stack, sizes, stream);
      if (rc) return rc;
      const long long cnt = (long long)B * (L.h[l] + ((L.stack && l >= 9 && l <= 12) ? 1 : 0)) * L.w[l] * kConvs[l].cout;
      CTPN_CUDA(cudaMemsetAsync(n->absmax_dev, 0, sizeof(unsigned), st));
      absmax_f16_kernel<<<1184, 256, 0, st>>>((const __half *)(ws + L.act[l]), cnt, n->absmax_dev);
      CTPN_LAUNCH_CHECK();
      unsigned bits = 0;
      CTPN_CUDA(cudaMemcpyAsync(&bits, n->absmax_dev, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
      CTPN_CUDA(cudaStreamSynchronize(st));
      float mx;
      memcpy(&mx, &bits, sizeof(float));
      CTPN_REQUIRE(mx == mx, "calibration: layer %s produced NaN", kConvs[l].name);
      if (std::isinf(mx) || mx >= 60000.f) {     // the fp16 plane saturated: shrink and retry
        CTPN_REQUIRE(attempt < 6, "calibration: activations of %s exceed 65504 * 2^48", kConvs[l].name);
        s_try *= 1.f / 256.f;
        continue;
      }
      const float amax = std::max(mx / s_try, 1e-20f);           // max |activation| of this layer on the calibration batch
      n->act_max[l] = amax;
      n->act_s[l] = amax * s_try > 16384.f || s_try < 1.f ? exp2f(floorf(log2f(16384.f / amax))) : 1.f;
      n->act_t[l] = exp2f(floorf(log2f(448.f / amax)) - 2.f);    // two binades of headroom; beyond that e4m3 saturates (cross term only)
      break;
    }
    int rc = l == 0 ? conv1_1_tc_ragged(images, src_is_f32, n->lut, n->c11_w, n->c11_b, ws + L.act[0], B, h, w, 2, true, n->act_s[0],
                                        n->act_t[0], sizes, stream)
                    : run_layer_f16f8(n, l, in, ws + L.act[l], B, h, w, L.stack, sizes, stream);
    if (rc) return rc;
    h = L.h[l]; w = L.w[l];
  }
  n->calibrated = true;
  return CTPN_OK;
}

}  // namespace ctpn

extern "C" int ctpn_net_create(ctpn_net_t **net, int planes) {
  CTPN_REQUIRE(net, "ctpn_net_create: null pointer");
  CTPN_REQUIRE((planes >= 1 && planes <= 3) || planes == CTPN_ARITH_F16F8 || planes == CTPN_ARITH_BF16X3P,
               "ctpn_net_create: planes must be 1..3, CTPN_ARITH_F16F8 or CTPN_ARITH_BF16X3P (got %d)", planes);
  ctpn_net *n = new ctpn_net();
  n->f16f8 = planes == CTPN_ARITH_F16F8;
  n->promote = planes == CTPN_ARITH_BF16X3P;
  n->planes = n->f16f8 ? 2 : n->promote ? 3 : planes;
  *net = n;
  return CTPN_OK;
}

extern "C" int ctpn_net_destroy(ctpn_net_t *net) {
  if (!net) return CTPN_OK;
  free_device(net);
  delete net;
  return CTPN_OK;
}

extern "C" int ctpn_net_set_option(ctpn_net_t *net, const char *key, int value) {
  CTPN_REQUIRE(net && key, "ctpn_net_set_option: null pointer");
  if (!strcmp(key, "keep_activations")) net->keep = value != 0;
  else if (!strcmp(key, "recalibrate")) net->calibrated = false;
#ifdef CTPN_DEBUG   // float32 SIMT reference kernels: test library only
  else if (!strcmp(key, "conv_simt")) net->conv_simt = value != 0;
  else if (!strcmp(key, "conv1_simt")) net->conv1_simt = value != 0;
#endif
  else { set_error("ctpn_net_set_option: unknown key '%s'", key); return CTPN_ERR_INVALID; }
  return CTPN_OK;
}

extern "C" int ctpn_net_set_weight(ctpn_net_t *net, const char *name, const float *data_host, size_t count) {
  CTPN_REQUIRE(net && name && data_host, "ctpn_net_set_weight: null pointer");
  net->host[name].assign(data_host, data_host + count);
  net->dirty = true;
  return CTPN_OK;
}

extern "C" int ctpn_net_feature_hw(int H, int W, int *fh, int *fw) {
  CTPN_REQUIRE(fh && fw && H >= 16 && W >= 16, "ctpn_net_feature_hw: image must be at least 16x16");
  *fh = H / 2 / 2 / 2 / 2;   // four VALID 2x2/2 pools: floor at every level
  *fw = W / 2 / 2 / 2 / 2;
  return CTPN_OK;
}

extern "C" size_t ctpn_net_workspace_bytes(const ctpn_net_t *net, int B, int H, int W) {
  if (!net || B <= 0 || H < 16 || W < 16) return 0;
  return net_layout(net, B, H, W).total;
}

// The network forward of a uniform batch (sizes = null) or of a ragged one (sizes = device int32 [B][2] image sizes on the
// canvas [B][H][W]): every stage gets the extents and stores zeros outside them, which the next 3x3 layer reads as padding.
static int net_forward(ctpn_net *net, const void *images, int src_is_f32, const int *sizes, int B, int H, int W,
                       float *cls_score_out, float *bbox_pred_out, void *workspace, size_t workspace_bytes, void *stream) {
#ifdef CTPN_DEBUG
  CTPN_REQUIRE(!sizes || !(net->conv_simt || net->conv1_simt), "ctpn_net_forward_ragged: the SIMT reference kernels take uniform batches only");
#endif
  int rc = finalize(net);
  if (rc) return rc;
  const NetLayout L = net_layout(net, B, H, W);
  if (workspace_bytes < L.total) {
    set_error("ctpn_net_forward: workspace %zu < %zu bytes", workspace_bytes, L.total);
    return CTPN_ERR_WORKSPACE;
  }
  char *ws = (char *)workspace;
  const int P = net->planes;
  net->taps.clear();
  if (net->f16f8) {
    // 2-unit arithmetic: conv1_1 and the thirteen 3x3 layers on F16F8 planes (calibrated on the first batch)
    if (!net->calibrated && (rc = calibrate_f16f8(net, images, src_is_f32, sizes, B, H, W, L, ws, stream))) return rc;
    int hh = H, ww = W;
    if ((rc = conv1_1_tc_ragged(images, src_is_f32, net->lut, net->c11_w, net->c11_b, ws + L.act[0], B, H, W, 2, true, net->act_s[0],
                                net->act_t[0], sizes, stream))) return rc;
    net->taps["conv1_1"] = Tap{ws + L.act[0], (long long)B * H * W, 64, true, net->act_s[0], net->act_t[0]};
    for (int l = 1; l < 14; ++l) {
      if (L.stack && l == 9)      // conv4_3 writes only the image rows of its stacked output: the pad rows must be zero
        CTPN_CUDA(cudaMemsetAsync(ws + L.act[9], 0, (size_t)P * B * (L.h[9] + 1) * L.w[9] * kConvs[9].cout * 2, (cudaStream_t)stream));
      if ((rc = run_layer_f16f8(net, l, ws + L.act[l - 1], ws + L.act[l], B, hh, ww, L.stack, sizes, stream))) return rc;
      hh = L.h[l]; ww = L.w[l];
      const ConvSpec &s = kConvs[l];
      const bool stacked = L.stack && l >= 9 && l <= 12;
      net->taps[s.pool ? std::string(s.name) + "+pool" : std::string(s.name)] =
          Tap{ws + L.act[l], (long long)B * hh * ww, s.cout, true, l == 13 ? 0.f : net->act_s[l], l == 13 ? 0.f : net->act_t[l],
              stacked ? hh : 0, stacked ? ww : 0};
    }
  }
  auto conv1 = [&](const void *src, int f32, const float *lut, const float *w, const float *b, void *out, int B_, int H_, int W_, int P_,
                   void *st) {
#ifdef CTPN_DEBUG
    if (net->conv_simt || net->conv1_simt) return ctpn_conv1_1(src, f32, lut, w, b, out, B_, H_, W_, P_, st);
#endif
    return conv1_1_tc_ragged(src, f32, lut, w, b, out, B_, H_, W_, P_, false, 1.f, 1.f, sizes, st);
  };
  // 3x3 layers pass the extents (output level `lvl`); the 1x1 matmuls run on the whole canvas (sizes = null)
  auto conv3 = [&](const void *in, const void *w, const float *b, void *out, int B_, int H_, int W_, int cin, int cout, int taps, int P_,
                   int flags, const int *sz, int lvl, void *st) {
#ifdef CTPN_DEBUG
    if (net->conv_simt) return ctpn_conv3x3_simt(in, w, b, out, B_, H_, W_, cin, cout, taps, P_, flags, st);
#endif
    return conv3x3_ragged(in, w, b, out, B_, H_, W_, cin, cout, taps, P_, flags, sz, lvl, st);
  };
  const int pf = net->promote ? CTPN_F_PROMOTE : 0;     // CTPN_ARITH_BF16X3P: every conv_tc layer below
  if (!net->f16f8) {
  if ((rc = conv1(images, src_is_f32, net->lut, net->c11_w, net->c11_b, ws + L.act[0], B, H, W, P, stream))) return rc;
  net->taps["conv1_1"] = Tap{ws + L.act[0], (long long)B * H * W, 64, true};
  int h = H, w = W;
  for (int l = 1; l < 14; ++l) {
    const ConvSpec &s = kConvs[l];
    int flags = CTPN_F_RELU | (s.pool ? CTPN_F_POOL : 0) | pf;
    const bool stacked = L.stack && l >= 9 && l <= 12;
    if (stacked) flags |= CTPN_F_STACK_OUT;
    if (L.stack && l >= 10) flags |= CTPN_F_STACK_IN;
    if (L.stack && l == 9)      // conv4_3 writes only the image rows of its stacked output: the pad rows must be zero
      CTPN_CUDA(cudaMemsetAsync(ws + L.act[9], 0, (size_t)P * B * (L.h[9] + 1) * L.w[9] * kConvs[9].cout * 2, (cudaStream_t)stream));
    if ((rc = conv3(ws + L.act[l - 1], net->conv_w[l], net->conv_b[l], ws + L.act[l], B, h, w, s.cin, s.cout, 9, P, flags, sizes,
                    out_level(l), stream))) return rc;
    h = L.h[l]; w = L.w[l];
    net->taps[s.pool ? std::string(s.name) + "+pool" : std::string(s.name)] =
        Tap{ws + L.act[l], (long long)B * h * w, s.cout, true, 0.f, 0.f, stacked ? h : 0, stacked ? w : 0};
  }
  }
  const int M = B * L.fh * L.fw;
  auto gemm = [&](const void *in, const void *w, const float *b, void *out, int cin, int cout, int flags) {
    return conv3(in, w, b, out, 1, 1, M, cin, cout, 1, P, flags, nullptr, 0, stream);
  };
  if ((rc = gemm(ws + L.act[13], net->xproj_w, net->xproj_b, ws + L.xproj, 512, 1024, CTPN_F_OUT_F32 | pf))) return rc;
  net->taps["xproj"] = Tap{ws + L.xproj, M, 1024, false};
  if ((rc = bilstm_ragged((const float *)(ws + L.xproj), net->wh_fw, net->wh_bw, ws + L.act[14], B * L.fh, L.fw, P, sizes, L.fh, stream))) return rc;
  net->taps["lstm_out"] = Tap{ws + L.act[14], M, 256, true};
  if ((rc = gemm(ws + L.act[14], net->fc_w, net->fc_b, ws + L.act[15], 256, 512, pf))) return rc;
  net->taps["lstm_o"] = Tap{ws + L.act[15], M, 512, true};
  if ((rc = gemm(ws + L.act[15], net->head_w, net->head_b, ws + L.heads, 512, 64, CTPN_F_OUT_F32 | pf))) return rc;
  const long long tot = (long long)M * 64;
  split_heads_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const float *)(ws + L.heads), M, cls_score_out, bbox_pred_out);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

extern "C" int ctpn_net_forward(ctpn_net_t *net, const void *images, int src_is_f32, int B, int H, int W,
                                float *cls_score_out, float *bbox_pred_out, void *workspace, size_t workspace_bytes,
                                void *stream) {
  CTPN_REQUIRE(net && images && cls_score_out && bbox_pred_out && workspace, "ctpn_net_forward: null pointer");
  CTPN_REQUIRE(B > 0 && H >= 16 && W >= 16, "ctpn_net_forward: bad shape B=%d H=%d W=%d", B, H, W);
  return net_forward(net, images, src_is_f32, nullptr, B, H, W, cls_score_out, bbox_pred_out, workspace, workspace_bytes, stream);
}

extern "C" int ctpn_net_forward_ragged(ctpn_net_t *net, const void *images, int src_is_f32, const int *sizes, int B, int H, int W,
                                       float *cls_score_out, float *bbox_pred_out, void *workspace, size_t workspace_bytes,
                                       void *stream) {
  CTPN_REQUIRE(net && images && sizes && cls_score_out && bbox_pred_out && workspace, "ctpn_net_forward_ragged: null pointer");
  CTPN_REQUIRE(B > 0 && H >= 16 && W >= 16, "ctpn_net_forward_ragged: bad shape B=%d H=%d W=%d", B, H, W);
  return net_forward(net, images, src_is_f32, sizes, B, H, W, cls_score_out, bbox_pred_out, workspace, workspace_bytes, stream);
}

extern "C" int ctpn_net_debug_tap(ctpn_net_t *net, const char *name, float *out_f32, size_t capacity, size_t *count,
                                  void *stream) {
  CTPN_REQUIRE(net && name && count, "ctpn_net_debug_tap: null pointer");
  auto it = net->taps.find(name);
  CTPN_REQUIRE(it != net->taps.end(), "ctpn_net_debug_tap: no activation named '%s' (run a forward first)", name);
  const Tap &t = it->second;
  const long long n = t.pixels * t.channels;
  *count = (size_t)n;
  if (!out_f32) return CTPN_OK;
  CTPN_REQUIRE(capacity >= (size_t)n, "ctpn_net_debug_tap: buffer too small (%zu < %lld)", capacity, n);
  if (t.planes && t.q_s > 0.f) {
    const long long stored = t.stack_h ? n / t.stack_h * (t.stack_h + 1) : n;      // elements per plane incl. pad rows
    f16f8_to_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const __half *)t.ptr, (const uint8_t *)t.ptr + stored * 2, n,
                                                                                       t.channels, t.q_s, t.q_t, t.stack_h, t.stack_w, out_f32);
    CTPN_LAUNCH_CHECK();
  } else if (t.planes) {
    const long long stored = t.stack_h ? n / t.stack_h * (t.stack_h + 1) : n;      // elements per plane incl. pad rows
    planes_to_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)t.ptr, n, stored, net->planes, t.channels,
                                                                                        t.stack_h, t.stack_w, out_f32);
    CTPN_LAUNCH_CHECK();
  } else {
    CTPN_CUDA(cudaMemcpyAsync(out_f32, t.ptr, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  }
  return CTPN_OK;
}
