// conv1_1 on the tensor cores: 3 -> 64 channels, K = 27 (padded to 32), uint8 / float32 image in, bf16 planes out.
//
// The layer is HBM-write bound (3 B in, 64 * P * 2 B out per pixel); the float32 SIMT version (conv_simt.cu) spends
// 1728 FMAs per pixel and reaches only a third of that bound.  Here the im2col tile is built IN SHARED MEMORY:
//   * 4 builder warps (thread = pixel of a 16 x 8 patch) gather the 27 mean-subtracted inputs of their pixel from a
//     small staged image patch, split them into P bf16 planes and write one K-major 128-byte row per plane in the
//     128B-swizzled wgmma layout (only the first 64 bytes = 32 k-values are ever read),
//   * k = 27 of the padded K = 32 carries the bias (A holds the constant 1 there), so the epilogue has no bias add,
//   * two consumer warpgroups issue 2 (k-slices) x {1,3,6} (plane pairs) wgmma of shape 64 x 64 x 16 each per tile
//     against the CTA-resident weight tile (built once from the float32 HWIO weights),
//   * the same 8 warps (thread = pixel, one 32-channel half per set of 4 warps) then do ReLU + plane split and store
//     through a float32 staging buffer and the same shared-memory transpose as conv_tc -- the epilogue, not the MMAs,
//     paces this layer.
// Accumulators (main + cross, see conv_tc.cu) live in registers.  Each builder group owns kSPG A stages (two for P <= 2),
// so it builds its next tile while the consumers are still on the previous one.
// Numerics: operands carry P bf16 planes like every other tensor-core layer (planes=3 is float32-equivalent).
// Reference semantics: lib/networks/network.py:160-183 (conv1_1), lib/fast_rcnn/test.py:8-9 (mean subtraction).
#include <mutex>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace ctpn {

#ifdef CTPN_DEBUG
#define C1_DBG(p, bit) (((p).debug & (bit)) != 0)
#else
#define C1_DBG(p, bit) false
#endif


constexpr int kC1tThreads = 512;          // warps 0-7: two builder groups, warps 8-15: two MMA + epilogue warpgroups
constexpr int kC1tTileBytes = 128 * 128;  // one plane of the A tile (128 pixels x 128-byte rows)
constexpr int kC1tPatch = 3 * 18 * 40;     // floats per staged input patch

struct Conv1TcParams {
  const void *src;
  const float *lut, *w, *bias;
  __nv_bfloat16 *out;
  int B, H, W, src_is_f32;
  int tiles_x, tiles_y, total_tiles;
  int debug;   // test library only (CTPN_C1_DEBUG bits): 1 skip patch staging, 2 skip tile build, 4 skip stores, 8 skip epilogue math
  long long plane_stride;
  float out_s, out_t, out_rs;    // OUTQ: F16F8 output quantisation (common.cuh), out_rs = 2^11 * out_t / out_s
  const int *sizes;              // ragged batch: device int32 [B][2] image sizes (h, w); pixels outside are SAME padding
};

// extent of image b: its (h, w) from sizes clamped to the canvas, or the canvas
__device__ __forceinline__ void c1_extent(const Conv1TcParams &p, int b, int &eh, int &ew) {
  eh = p.H; ew = p.W;
  if (p.sizes) {
    eh = min(eh, __ldg(p.sizes + 2 * b));
    ew = min(ew, __ldg(p.sizes + 2 * b + 1));
  }
}

// OUTQ = 1: the output is written in the F16F8 activation format (fp16 plane + e4m3 value / residual plane) for a
// conv1_2 that runs in the 2-unit arithmetic; the layer itself still multiplies P bf16 planes (K = 27: the MMAs are free).
template <int P, int OUTQ>
__global__ void __launch_bounds__(kC1tThreads, 1)
conv1_tc_kernel(const Conv1TcParams p) {
  using namespace ptx;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  constexpr int kSPG = P <= 2 ? 2 : 1;                        // A stages per builder group
  constexpr int kStages = 2 * kSPG;
  const uint32_t a0 = (raw + 1023u) & ~1023u;                 // A tiles: [kStages][P planes][16 KB]
  const uint32_t b0 = a0 + (uint32_t)kStages * P * kC1tTileBytes;   // weights: [P planes][64 rows x 128 B]
  uint8_t *base = smem_raw + (a0 - raw);
  uint8_t *bsm = base + kStages * P * kC1tTileBytes;
  // input patches (two per builder group): [3 channels][18 rows][40]: a row pitch of 40 floats makes the builders' gather
  // (lanes = 4 tile rows x 8 tile columns) hit 32 distinct banks
  float *patch = reinterpret_cast<float *>(bsm + P * 64 * 128);
  float *lut_s = patch + 4 * kC1tPatch;                                 // [256][3] mean-subtraction table
  float *epi = lut_s + 768;                                             // float32 staging [2 chunks][128 pixels][32 channels]
  uint64_t *bars = reinterpret_cast<uint64_t *>(epi + 2 * 128 * 32);
  const uint32_t fullA = smem_u32(bars), emptyA = fullA + 32;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < 4; ++i) {
      mbar_init(fullA + 8 * i, 128);     // every builder thread arrives
      mbar_init(emptyA + 8 * i, 2);      // the two consumer warpgroups, once their MMAs have completed
    }
    fence_mbar_init();
  }
  if (!p.src_is_f32)
    for (int i = threadIdx.x; i < 768; i += kC1tThreads) lut_s[i] = p.lut[i];
  // resident weight tile: row = cout, k-major, bf16 planes, 128B swizzle (chunk ^= row & 7); k >= 27 is zero
  for (int i = threadIdx.x; i < 64 * 4; i += kC1tThreads) {
    const int co = i >> 2, chunk = i & 3;
    uint32_t pk[3][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float v[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int k = chunk * 8 + j * 2 + e;
        v[e] = k < 27 ? p.w[k * 64 + co] : (k == 27 ? p.bias[co] : 0.f);   // k = 27: bias row (A carries a 1 there)
      }
      uint32_t t[P];
      split_planes2<P>(v[0], v[1], t);
#pragma unroll
      for (int pl = 0; pl < P; ++pl) pk[pl][j] = t[pl];
    }
#pragma unroll
    for (int pl = 0; pl < P; ++pl)
      *reinterpret_cast<uint4 *>(bsm + pl * 64 * 128 + co * 128 + ((chunk ^ (co & 7)) << 4)) = make_uint4(pk[pl][0], pk[pl][1], pk[pl][2], pk[pl][3]);
  }
  fence_proxy_async();
  __syncthreads();
  const int tiles_per_img = p.tiles_x * p.tiles_y;

  if (warp < 8) {
    // ===== im2col builders: two groups of 4 warps; group g owns stage g and builds every other tile of this CTA,
    // so two tiles are in flight and the global-load latency of the patch staging is hidden.  thread = pixel m =====
    const int grp = warp >> 2;
    const int m = (warp & 3) * 32 + lane, th = m >> 3, tw = m & 7;
    // The raw inputs of the NEXT tile's patch pixels (this thread stages patch pixels m and m + 128 of 180) are
    // fetched into registers while the current tile is being built, so the global-load latency is off the
    // per-tile critical path of the group.
    const unsigned tpi = (unsigned)tiles_per_img, tx = (unsigned)p.tiles_x;
    uint32_t raw[2][3];
    unsigned valid = 0;
    auto fetch = [&](int tile) {
      valid = 0;
      if (tile >= p.total_tiles) return;
      const unsigned b = (unsigned)tile / tpi, r = (unsigned)tile % tpi;
      const int y0 = (int)(r / tx) * 16, x0 = (int)(r % tx) * 8;
      int eh, ew;
      c1_extent(p, (int)b, eh, ew);
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int i = m + u * 128;
        const int xx = i % 10, yy = i / 10;
        const int gx = x0 + xx - 1, gy = y0 + yy - 1;
        if (i < 180 && gx >= 0 && gx < ew && gy >= 0 && gy < eh && !C1_DBG(p, 1)) {
          const size_t off = (((size_t)b * p.H + gy) * p.W + gx) * 3;
          if (p.src_is_f32) {
            const float *q = reinterpret_cast<const float *>(p.src) + off;
            raw[u][0] = __float_as_uint(q[0]); raw[u][1] = __float_as_uint(q[1]); raw[u][2] = __float_as_uint(q[2]);
          } else {
            const uint8_t *q = reinterpret_cast<const uint8_t *>(p.src) + off;
            raw[u][0] = q[0]; raw[u][1] = q[1]; raw[u][2] = q[2];
          }
          valid |= 1u << u;
        }
      }
    };
    fetch(blockIdx.x + grp * gridDim.x);
    int n = 0;
    for (int tile = blockIdx.x + grp * gridDim.x; tile < p.total_tiles; tile += 2 * gridDim.x, ++n) {
      const int s = grp * kSPG + n % kSPG;
      const uint32_t ph = (uint32_t)(n / kSPG) & 1u;
      // two patches per group: a fast warp may stage tile n + 1 while a slow one still gathers from tile n's patch;
      // it cannot get to tile n + 2 before the group barrier of tile n + 1, which the slow warp reaches after tile n
      float *pt = patch + (grp * 2 + (n & 1)) * kC1tPatch;
      // stage the 18 x 10 x 3 mean-subtracted input patch (zero outside the image: SAME padding of the blob; in a ragged batch
      // the canvas outside the image's extent is never read)
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int i = m + u * 128;
        if (i < 180) {
          const int xx = i % 10, yy = i / 10;
          float v0 = 0.f, v1 = 0.f, v2 = 0.f;
          if ((valid >> u) & 1u) {
            if (p.src_is_f32) {
              v0 = __uint_as_float(raw[u][0]); v1 = __uint_as_float(raw[u][1]); v2 = __uint_as_float(raw[u][2]);
            } else {
              v0 = lut_s[raw[u][0] * 3 + 0]; v1 = lut_s[raw[u][1] * 3 + 1]; v2 = lut_s[raw[u][2] * 3 + 2];
            }
          }
          pt[(0 * 18 + yy) * 40 + xx] = v0;
          pt[(1 * 18 + yy) * 40 + xx] = v1;
          pt[(2 * 18 + yy) * 40 + xx] = v2;
        }
      }
      fetch(tile + 2 * gridDim.x);            // next tile of this group: loads stay in flight during the build
      mbar_wait(emptyA + 8 * s, ph ^ 1u);     // MMAs that read this A stage are done
      if (grp == 0) asm volatile("bar.sync 1, 128;" ::: "memory");     // the four warps of this builder group
      else asm volatile("bar.sync 2, 128;" ::: "memory");
      uint8_t *arow = base + s * P * kC1tTileBytes + m * 128;
#pragma unroll
      for (int chunk = 0; chunk < (C1_DBG(p, 2) ? 0 : 4); ++chunk) {
        uint32_t pk[3][4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float v[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int k = chunk * 8 + j * 2 + e;       // k = (ky * 3 + kx) * 3 + c
            v[e] = k < 27 ? pt[((k % 3) * 18 + th + k / 9) * 40 + tw + (k / 3) % 3] : (k == 27 ? 1.f : 0.f);
          }
          uint32_t t[P];
          split_planes2<P>(v[0], v[1], t);
#pragma unroll
          for (int pl = 0; pl < P; ++pl) pk[pl][j] = t[pl];
        }
#pragma unroll
        for (int pl = 0; pl < P; ++pl)
          *reinterpret_cast<uint4 *>(arow + pl * kC1tTileBytes + ((chunk ^ (m & 7)) << 4)) = make_uint4(pk[pl][0], pk[pl][1], pk[pl][2], pk[pl][3]);
      }
      fence_proxy_async();                   // generic-proxy writes -> visible to the tensor core (async proxy)
      mbar_arrive(fullA + 8 * s);
    }
  } else {
    // ===== consumers: warpgroup wg multiplies tile rows [64 wg, 64 wg + 64) against the 64 output channels; then the
    // epilogue with thread = pixel m (warps 8-11 take channels 0-31, 12-15 channels 32-63) =====
    const int wg = (warp >> 2) - 2;
    const int cw = warp - 8, chunk = cw >> 2, quarter = cw & 3;
    const int m = quarter * 32 + lane, th = m >> 3, tw = m & 7;
    const int frow = wg * 64 + (warp & 3) * 16 + (lane >> 2);     // accumulator fragment rows frow, frow + 8
    constexpr uint32_t kHi = gmma_desc_hi(1024);
    const uint32_t b_lo = gmma_desc_lo(b0);
    float accm[32], accc[32];
    // the warp's own 32 staging rows double as its store-transpose block once they have been read
    uint4 *stage_w = reinterpret_cast<uint4 *>(epi + chunk * 4096 + quarter * 1024);
    int n = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++n) {
      // tile n of this CTA was built by group n & 1 as its (n >> 1)-th tile
      const int s = (n & 1) * kSPG + (n >> 1) % kSPG;
      const uint32_t ph = (uint32_t)((n >> 1) / kSPG) & 1u;
      const unsigned b = (unsigned)tile / (unsigned)tiles_per_img, r = (unsigned)tile % (unsigned)tiles_per_img;
      const int y = (int)(r / (unsigned)p.tiles_x) * 16 + th, x = (int)(r % (unsigned)p.tiles_x) * 8 + tw;
      const bool ok = y < p.H && x < p.W;
      int eh, ew;
      c1_extent(p, (int)b, eh, ew);
      const bool live = y < eh && x < ew;     // false: ragged padding, stored as zero (the bias row would make it ReLU(bias))
      const long long pix = ((long long)b * p.H + y) * p.W + x;
      const unsigned okmask = __ballot_sync(0xffffffffu, ok);
      long long spix[4];
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const long long hi = __shfl_sync(0xffffffffu, (int)(pix >> 32), it * 8 + (lane >> 2));
        const unsigned lo = __shfl_sync(0xffffffffu, (unsigned)(pix & 0xffffffffll), it * 8 + (lane >> 2));
        spix[it] = (hi << 32) | lo;
      }
      mbar_wait(fullA + 8 * s, ph);
      const uint32_t a_lo = gmma_desc_lo(a0 + s * P * kC1tTileBytes + wg * 64 * 128);
      wgmma_fence();
#pragma unroll
      for (int i = 0; i < P; ++i)
#pragma unroll
        for (int j = 0; j < P - i; ++j)
#pragma unroll
          for (int k = 0; k < 2; ++k) {   // K = 32 (27 real taps): two 16-wide slices
            const uint64_t da = ((uint64_t)kHi << 32) | (a_lo + i * (kC1tTileBytes >> 4) + 2u * k);
            const uint64_t db = ((uint64_t)kHi << 32) | (b_lo + j * ((64 * 128) >> 4) + 2u * k);
            if (i + j == 0) wgmma_bf16(accm, da, db, (uint32_t)k);
            else wgmma_bf16(accc, da, db, (k == 0 && i == 0 && j == 1) ? 0u : 1u);
          }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(accm);
      if (P > 1) wgmma_fence_regs(accc);
      if ((threadIdx.x & 127) == 0) mbar_arrive(emptyA + 8 * s);
      if (P > 1) {
#pragma unroll
        for (int i = 0; i < 32; ++i) accm[i] = accm[i] + accc[i];
      }
      named_sync(3, 256);             // the previous tile's staging rows have been read and stored
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int q = 2 * (j & 3) + ((lane & 3) >> 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = frow + 8 * h;
          *reinterpret_cast<float2 *>(epi + (j >> 2) * 4096 + row * 32 + ((q ^ (row & 7)) << 2) + 2 * (lane & 1)) =
              make_float2(accm[4 * j + 2 * h], accm[4 * j + 2 * h + 1]);
        }
      }
      named_sync(3, 256);
      if (!C1_DBG(p, 8)) {
        float v[32];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 t = *reinterpret_cast<const float4 *>(epi + chunk * 4096 + m * 32 + ((q ^ (m & 7)) << 2));
          v[4 * q + 0] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
        }
        if (!live) {
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = 0.f;
        }
        // the bias came in through the tensor core (k = 27 row of the weight tile x the builders' constant 1)
        if (OUTQ) {
          uint32_t wh[16], wq[16];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float v0 = fmaxf(v[4 * i], 0.f), v1 = fmaxf(v[4 * i + 1], 0.f), v2 = fmaxf(v[4 * i + 2], 0.f), v3 = fmaxf(v[4 * i + 3], 0.f);
            f16f8_quad(v0, v1, v2, v3, p.out_s, p.out_t, p.out_rs, wh[2 * i], wh[2 * i + 1], wq[i], wq[8 + i]);
          }
#pragma unroll
          for (int pl = 0; pl < 2; ++pl) {
            __syncwarp();
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const uint4 val = pl == 0 ? make_uint4(wh[4 * q], wh[4 * q + 1], wh[4 * q + 2], wh[4 * q + 3])
                                        : make_uint4(wq[4 * q], wq[4 * q + 1], wq[4 * q + 2], wq[4 * q + 3]);
              stage_w[lane * 4 + (q ^ ((lane >> 1) & 3))] = val;
            }
            __syncwarp();
            // plane 0: 32 fp16 = 64 contiguous bytes per pixel; plane 1: values at +chunk*32, residuals at +64+chunk*32 of
            // the pixel's single 128-byte block (Cout = 64)
            uint8_t *obase = reinterpret_cast<uint8_t *>(p.out) + (long long)pl * p.plane_stride * 2;
            const int j = lane & 3;
            const int off = pl == 0 ? chunk * 64 + j * 16 : chunk * 32 + (j >> 1) * 64 + (j & 1) * 16;
#pragma unroll
            for (int it = 0; it < 4; ++it) {
              const int pp = it * 8 + (lane >> 2);
              const uint4 val = stage_w[pp * 4 + (j ^ ((pp >> 1) & 3))];
              if (((okmask >> pp) & 1u) && !C1_DBG(p, 4)) *reinterpret_cast<uint4 *>(obase + spix[it] * 128 + off) = val;
            }
          }
        } else {
        uint32_t w[P][16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          uint32_t t[P];
          split_planes2<P>(fmaxf(v[2 * i], 0.f), fmaxf(v[2 * i + 1], 0.f), t);
#pragma unroll
          for (int pl = 0; pl < P; ++pl) w[pl][i] = t[pl];
        }
#pragma unroll
        for (int pl = 0; pl < P; ++pl) {
          __syncwarp();
#pragma unroll
          for (int q = 0; q < 4; ++q) stage_w[lane * 4 + (q ^ ((lane >> 1) & 3))] = make_uint4(w[pl][4 * q], w[pl][4 * q + 1], w[pl][4 * q + 2], w[pl][4 * q + 3]);
          __syncwarp();
          __nv_bfloat16 *obase = p.out + (long long)pl * p.plane_stride + chunk * 32 + (lane & 3) * 8;
#pragma unroll
          for (int it = 0; it < 4; ++it) {
            const int pp = it * 8 + (lane >> 2);
            const uint4 val = stage_w[pp * 4 + ((lane & 3) ^ ((pp >> 1) & 3))];
            if (((okmask >> pp) & 1u) && !C1_DBG(p, 4)) *reinterpret_cast<uint4 *>(obase + spix[it] * 64) = val;
          }
        }
        }
      }
    }
  }
}

template <int P, int OUTQ = 0>
static int launch_conv1_tc(Conv1TcParams &p, cudaStream_t st) {
  const size_t smem = 1024 + (size_t)(P <= 2 ? 4 : 2) * P * kC1tTileBytes + (size_t)P * 64 * 128 +
                      (4 * kC1tPatch + 768 + 2 * 128 * 32) * sizeof(float) + 64;
  constexpr int kMaxDevices = 64;
  static std::mutex mu;
  static int sm_count[kMaxDevices];      // per device: SM count (0 = attribute not set yet)
  int dev = 0;
  CTPN_CUDA(cudaGetDevice(&dev));
  CTPN_REQUIRE(dev >= 0 && dev < kMaxDevices, "ctpn_conv1_1_tc: device index %d not supported", dev);
  int sms;
  {
    std::lock_guard<std::mutex> lock(mu);
    if (sm_count[dev] == 0) {
      CTPN_CUDA(cudaFuncSetAttribute(conv1_tc_kernel<P, OUTQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      CTPN_CUDA(cudaDeviceGetAttribute(&sm_count[dev], cudaDevAttrMultiProcessorCount, dev));
    }
    sms = sm_count[dev];
  }
  const int grid = p.total_tiles < sms ? p.total_tiles : sms;
  ProfScope prof("conv1_1", 2.0 * p.B * p.H * p.W * 27.0 * 64.0, st);
  conv1_tc_kernel<P, OUTQ><<<grid, kC1tThreads, smem, st>>>(p);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

}  // namespace ctpn

int ctpn::conv1_1_tc_ragged(const void *src, int src_is_f32, const float *lut, const float *w_hwio, const float *bias,
                            void *out_planes, int B, int H, int W, int planes, bool outq, float out_s, float out_t,
                            const int *sizes, void *stream) {
  CTPN_REQUIRE(src && w_hwio && bias && out_planes, "ctpn_conv1_1_tc: null pointer");
  CTPN_REQUIRE(src_is_f32 || lut, "ctpn_conv1_1_tc: uint8 input needs the mean-subtraction LUT");
  CTPN_REQUIRE(B > 0 && H > 0 && W > 0, "ctpn_conv1_1_tc: bad shape");
  CTPN_REQUIRE(planes >= 1 && planes <= 3, "ctpn_conv1_1_tc: planes must be 1..3");
  Conv1TcParams p;
  p.src = src; p.lut = lut; p.w = w_hwio; p.bias = bias; p.out = (__nv_bfloat16 *)out_planes;
  p.B = B; p.H = H; p.W = W; p.src_is_f32 = src_is_f32;
  p.tiles_x = ceil_div(W, 8); p.tiles_y = ceil_div(H, 16);
  const long long total = (long long)B * p.tiles_x * p.tiles_y;
  CTPN_REQUIRE(total < (1ll << 31), "ctpn_conv1_1_tc: too many tiles");
  p.total_tiles = (int)total;
  p.plane_stride = (long long)B * H * W * 64;
  p.out_s = p.out_t = p.out_rs = 1.f;
  p.sizes = sizes;
  if (outq) {
    CTPN_REQUIRE(out_s > 0.f && out_t > 0.f, "ctpn_conv1_1_tc_f16f8: scales must be positive");
    p.out_s = out_s; p.out_t = out_t; p.out_rs = kResidualGain * out_t / out_s;
  }
#ifdef CTPN_DEBUG
  static const int dbg = [] { const char *e = getenv("CTPN_C1_DEBUG"); return e ? atoi(e) : 0; }();
  p.debug = dbg;
#else
  p.debug = 0;
#endif
  cudaStream_t st = (cudaStream_t)stream;
  if (outq) return launch_conv1_tc<2, 1>(p, st);
  if (planes == 1) return launch_conv1_tc<1>(p, st);
  if (planes == 2) return launch_conv1_tc<2>(p, st);
  return launch_conv1_tc<3>(p, st);
}

using namespace ctpn;

extern "C" int ctpn_conv1_1_tc(const void *src, int src_is_f32, const float *lut, const float *w_hwio, const float *bias,
                               void *out_planes, int B, int H, int W, int planes, void *stream) {
  return conv1_1_tc_ragged(src, src_is_f32, lut, w_hwio, bias, out_planes, B, H, W, planes, false, 1.f, 1.f, nullptr, stream);
}

extern "C" int ctpn_conv1_1_tc_f16f8(const void *src, int src_is_f32, const float *lut, const float *w_hwio, const float *bias,
                                     void *out_planes, int B, int H, int W, float out_s, float out_t, void *stream) {
  return conv1_1_tc_ragged(src, src_is_f32, lut, w_hwio, bias, out_planes, B, H, W, 2, true, out_s, out_t, nullptr, stream);
}
