// 3x3 SAME convolution / 1x1 matmul on bf16 "planes" with Hopper warpgroup MMAs (wgmma).
//
// Implicit GEMM: M = 128 output pixels (a 16 x 8 patch of one image per CTA tile), N = BN output
// channels, K = taps * Cin in blocks of 64 channels.
//   * A operand: per channel block ONE 4-D TMA box load brings the (16+2) x (8+2) x 64 halo patch of the
//     NHWC input into shared memory (128-byte swizzle; out-of-image elements are zero-filled by the TMA
//     unit = SAME padding and ragged edges for free).  The nine filter taps are then served as nine
//     shifted VIEWS of that one patch: the wgmma shared-memory descriptor starts at halo row
//     (ky * 10 + kx) and steps 10 rows between its 8-row groups (tile row th <-> halo row th + ky).  The
//     tensor core applies the 128B swizzle to the absolute shared-memory address, so un-aligned views of
//     a TMA-written buffer are consistent (checked by tests/probe_umma_view.py).  This cuts the
//     L2 -> SM traffic of A by 6.4x compared with one TMA load per tap.
//   * B operand: weights [P][Cout][taps][Cin] viewed as a 2-D K-major matrix, one 2-D TMA box per
//     (tap, channel block), in its own ring of stages.
//   * D: float32 accumulators in registers.  Two consumer warpgroups each own 64 of the 128 pixel rows (m64nBNk16
//     wgmma, or k32 for e4m3) and keep one group of MMAs in flight; a stage is released when its group completes.
//     With P > 1 planes the plane-0 x plane-0 products go to a "main" accumulator and all cross-plane
//     products to a second one (the tensor core truncates when adding into float32; see DESIGN.md).
//   * epilogue (thread = pixel): the combined accumulators go through a float32 staging buffer, 64 channels at a time ->
//     +bias -> ReLU -> optional fused 2x2 max-pool (warp shuffles: the window of a pixel lives in lanes l, l^1, l^8, l^9)
//     -> re-split into planes (cvt.rn.bf16x2.f32) -> transpose through swizzled shared memory -> 16-byte stores that
//     cover one pixel's 64 contiguous bytes with 4 lanes (or float32 output).
// Small and promoted 3x3 layers run as 2-CTA clusters that share every weight tile by TMA multicast (template parameter MC;
// CTPN_TC_MCAST=0 selects the single-CTA variant everywhere); large unpromoted ones run one CTA per SM (conv_tc_run).
// Persistent CTAs (one per SM), warp-specialised: warp 0 weight (B) producer, warp 1 activation (A) producer, warpgroups
// 1 and 2 MMAs, warpgroup 3 the epilogue: the MMA warpgroups hand each finished tile over through the staging buffer in
// 64-channel halves (an mbarrier full / empty pair) and start the next tile's MMAs while warpgroup 3 converts and stores
// it.  The promoted kernels (PR = 1: three accumulator arrays, no registers left for a fourth warpgroup) run the same
// epilogue on the two MMA warpgroups after each tile.  Reference: lib/networks/network.py:160-196.
#include <cuda.h>

#include <algorithm>
#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "tc_ptx.cuh"
#include "tma_host.cuh"

namespace ctpn {

// Ablation switches (skip loads / MMAs / stores) exist only in the test library (-DCTPN_DEBUG, env CTPN_TC_DEBUG); in
// the product build the tests below are compile-time false and the branches disappear.
#ifdef CTPN_DEBUG
#define CTPN_DBG(p, bit) (((p).debug & (bit)) != 0)
#else
#define CTPN_DBG(p, bit) false
#endif

struct ConvTcParams {
  int B, H, W, Cin, Cout, taps, planes, flags;
  int tiles_x, tiles_y, tiles_n, total_tiles;
  int m_tiles, total_units;  // pixel tiles; work units of the persistent loop (tiles, or with MC pairs of pixel tiles)
  int TH, TW, tw_log2;      // tile geometry (pixels); TH * TW == 128
  int PW;                   // halo patch width in pixels (= shared-memory rows per patch row)
  int patch_bytes;          // bytes of one plane's patch slot (1024-aligned)
  int patch_tx_bytes;       // bytes the TMA box actually transfers per plane
  int group_stride_bytes;   // wgmma stride between 8-row groups of the A view
  int cout_pad;
  int Ho, Wo;
  int stages_a, stages_b;
  int debug;                // test library only (CTPN_TC_DEBUG bits): 1 skip B loads, 2 skip A loads, 4 skip MMAs, 8 skip stores
  const float *bias;
  void *out;
  long long out_plane_stride;   // elements between output planes
  // F16F8 arithmetic (common.cuh): value = main * inv_main + cross * inv_cross; outputs are re-quantised as
  // h = fp16(v * out_s), e4m3(v * out_t), e4m3((v * out_s - h) * out_rs) with out_rs = 2^11 * out_t / out_s
  float inv_main, inv_cross, out_s, out_t, out_rs;
  // Row-stacked batches (CTPN_F_STACK_IN / _OUT): images stored as [B][H + 1][W][C] with one zero row after every image, so the
  // batch is ONE tall image for the tiling (a 37-row map wastes 23 % of its 16-row tiles, the 32 x 38-row stack 0 %) while the
  // zero rows keep the images' halos apart.  in_stack_h = rows per image incl. the pad row in the kernel's input frame (0 =
  // plain); out_rows = rows per image of the OUTPUT frame (Ho, or Ho + 1 when the output is stacked too).
  int in_stack_h, out_rows, out_stacked;
  // Ragged batches (ctpn_net_forward_ragged): ext = device int32 [ext_n][2] full-resolution image sizes (h, w), or null.  An
  // output pixel outside (h >> ext_shift, w >> ext_shift) of its image is stored as zero, so that the next 3x3 layer sees the
  // zeros as SAME padding.  Masking is value-only: loads, MMAs and the multicast pairing do not change.
  const int *ext;
  int ext_shift, ext_n;
  double work;              // algorithmic FLOPs of the call (profiling label only)
  int promote_every;        // test library only (CTPN_TC_PROMOTE): pipeline steps per promoted main chain (product: 1)
};

// warpgroup 0: producers (warp 0 weights, warp 1 activations); 1 and 2: MMAs; 3: epilogue.  PR = 1: 1 and 2 run MMAs and
// the epilogue.
// EW: the schedule with a dedicated epilogue warpgroup.  Not for the promoted kernels, and not at BN = 256: ptxas compiles a
// 512-thread kernel's m64n256 wgmma (128 accumulator registers + operands) against the launch's 128 registers per thread,
// whatever setmaxnreg grants the MMA warpgroups.
template <int BN, int PR> constexpr bool kEpiWarpgroup = !PR && BN <= 128;
template <int BN, int PR> constexpr int kTcThreads = kEpiWarpgroup<BN, PR> ? 512 : 384;
constexpr int kMaxStages = 8;
constexpr int kCtrlBytes = 8 * (4 * kMaxStages) + 16;   // the four stage rings' barriers + the epilogue handoff pair
constexpr int kEpiBytes = 2 * 128 * 32 * 4;        // float32 staging of two 32-channel chunks of the 128-pixel tile
constexpr int kXposeBytes = 4 * 512;               // epilogue warpgroup: a 512-byte store-transpose block per warp

// Where the epilogue thread of tile pixel m (lane = m & 31) writes, for pixel tile mt.  Warp-collective (ballot, shuffles).
struct EpiPixel {
  bool ok, live;        // ok: inside the output; live = false: stored as zero (a stacked pad row, or outside a ragged extent)
  int oy, ox;
  long long pix;        // output pixel index
  unsigned okmask;      // the warp's ok lanes
  long long spix[4];    // pixel of lane it * 8 + (lane >> 2): the transposed stores
};

__device__ __forceinline__ void epi_pixel(const ConvTcParams &p, int mt, int m, int lane, EpiPixel &e) {
  const int th = m >> p.tw_log2, tw = m & (p.TW - 1);
  const int tiles_per_img = p.tiles_x * p.tiles_y;
  const int b = mt / tiles_per_img, r = mt % tiles_per_img;
  const int y = (r / p.tiles_x) * p.TH + th, x = (r % p.tiles_x) * p.TW + tw;
  e.live = true;
  int ob = b;
  if (p.flags & CTPN_F_POOL) {
    e.oy = y >> 1; e.ox = x >> 1;
    e.ok = !(th & 1) && !(tw & 1) && e.oy < p.Ho && e.ox < p.Wo;
  } else {
    e.oy = y; e.ox = x;
    e.ok = y < p.H && x < p.W;
    if (p.in_stack_h) {       // stacked input: y runs over the whole stack (the kernel sees one image of B * in_stack_h rows)
      ob = y / p.in_stack_h;
      e.oy = y - ob * p.in_stack_h;
      e.live = e.oy < p.in_stack_h - 1;
      if (!p.out_stacked) e.ok = e.ok && e.live;
    }
  }
  if (p.ext) {     // ragged batch: zero outside the image's extent at the output level (with a pool: the whole window)
    const int ib = min(ob, p.ext_n - 1);
    e.live = e.live && e.oy < (__ldg(p.ext + 2 * ib) >> p.ext_shift) && e.ox < (__ldg(p.ext + 2 * ib + 1) >> p.ext_shift);
  }
  e.pix = ((long long)ob * p.out_rows + e.oy) * p.Wo + e.ox;
  // coalesced plane stores: the warp's 32-pixel x 32-channel block is transposed through shared memory so
  // that 4 consecutive lanes write the 64 contiguous bytes of one pixel (full 32-B sectors) instead of every
  // lane writing 16 B of its own pixel.  Lane l stores for pixels (l >> 2) + 8 * it, 16-byte chunk l & 3.
  e.okmask = __ballot_sync(0xffffffffu, e.ok);
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const long long hi = __shfl_sync(0xffffffffu, (int)(e.pix >> 32), it * 8 + (lane >> 2));
    const unsigned lo = __shfl_sync(0xffffffffu, (unsigned)(e.pix & 0xffffffffll), it * 8 + (lane >> 2));
    e.spix[it] = (hi << 32) | lo;
  }
}

// Each lane holds 64 bytes (w) of its own pixel; lane l stores 16-byte piece l & 3 of pixels (l >> 2) + 8 * it at
// obase + spix[it] * row_bytes.  small = 0: one 2-KB transpose block (the warp's 32 pixels at once); 1: a 512-byte block,
// 8 pixels per round.  16-byte pieces are XOR-swizzled by (row >> 1) & 3: conflict-free writes and reads.
__device__ __forceinline__ void store_transposed(uint4 *stage_w, const uint32_t (&w)[16], uint8_t *obase, long long row_bytes,
                                                 const EpiPixel &e, bool st_ok, bool small, int lane) {
  const int j = lane & 3;
  if (!small) {
    __syncwarp();     // previous readers of the staging block are done
#pragma unroll
    for (int q = 0; q < 4; ++q) stage_w[lane * 4 + (q ^ ((lane >> 1) & 3))] = make_uint4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
    __syncwarp();
    if (st_ok) {
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int pp = it * 8 + (lane >> 2);
        const uint4 val = stage_w[pp * 4 + (j ^ ((pp >> 1) & 3))];
        if ((e.okmask >> pp) & 1u) *reinterpret_cast<uint4 *>(obase + e.spix[it] * row_bytes) = val;
      }
    }
  } else {
    // lanes 8 it .. 8 it + 7 deposit their 64 bytes, all 32 lanes then store one 16-byte piece each
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      __syncwarp();
      if ((lane >> 3) == it) {
        const int row = lane & 7;
#pragma unroll
        for (int q = 0; q < 4; ++q) stage_w[row * 4 + (q ^ ((row >> 1) & 3))] = make_uint4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
      }
      __syncwarp();
      const int row = lane >> 2, pp = it * 8 + row;
      const uint4 val = stage_w[row * 4 + (j ^ ((row >> 1) & 3))];
      if (st_ok && ((e.okmask >> pp) & 1u)) *reinterpret_cast<uint4 *>(obase + e.spix[it] * row_bytes) = val;
    }
  }
}

// The epilogue of one 32-channel chunk (output channels c0 .. c0 + 31) of one pixel: v = the combined accumulators.
// +bias -> ReLU (unless the MMA warpgroups applied them: bias_relu = false) -> live mask -> optional fused 2x2 max-pool ->
// F16F8 / bf16 planes / float32 stores.
template <int P, int F8>
__device__ __forceinline__ void epi_chunk(const ConvTcParams &p, const EpiPixel &e, float (&v)[32], int c0, uint4 *stage_w,
                                          bool small, bool bias_relu, int lane) {
  const bool pool = (p.flags & CTPN_F_POOL) != 0, relu = (p.flags & CTPN_F_RELU) != 0;
  const bool out_f32 = (p.flags & CTPN_F_OUT_F32) != 0;
  if (bias_relu) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 bq = __ldg(reinterpret_cast<const float4 *>(p.bias + c0) + q);
      v[4 * q + 0] += bq.x;
      v[4 * q + 1] += bq.y;
      v[4 * q + 2] += bq.z;
      v[4 * q + 3] += bq.w;
    }
    if (relu) {
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], 0.f);
    }
  }
  if (!e.live) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = 0.f;
  }
  if (pool) {
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      v[i] = fmaxf(v[i], __shfl_xor_sync(0xffffffffu, v[i], 1));
      v[i] = fmaxf(v[i], __shfl_xor_sync(0xffffffffu, v[i], p.TW));
    }
  }
  if (F8 && pool && !out_f32 && !(p.flags & CTPN_F_OUT_BF16X2)) {
    // Pooled F16F8 output without staging: after the shuffles all four lanes of a 2x2 window (l, l^1, l^8, l^9) hold the
    // pooled value, so each takes one quarter (8 channels) of the chunk: a quarter of the conversions, and the four
    // lanes' stores form 64 contiguous bytes of the fp16 plane and 32 + 32 of the e4m3 plane (full sectors).
    const int j = (lane & 1) | ((lane >> 2) & 2);
    float x[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = j == 0 ? v[k] : j == 1 ? v[8 + k] : j == 2 ? v[16 + k] : v[24 + k];
    const bool okw = e.oy < p.Ho && e.ox < p.Wo;     // (pix already points into the stacked frame when out_rows = Ho + 1)
    uint4 hw;
    uint2 qv, qr;
    f16f8_quad(x[0], x[1], x[2], x[3], p.out_s, p.out_t, p.out_rs, hw.x, hw.y, qv.x, qr.x);
    f16f8_quad(x[4], x[5], x[6], x[7], p.out_s, p.out_t, p.out_rs, hw.z, hw.w, qv.y, qr.y);
    if (okw && c0 < p.Cout && !CTPN_DBG(p, 8)) {
      uint8_t *o0 = reinterpret_cast<uint8_t *>(p.out) + e.pix * p.Cout * 2;
      uint8_t *o1 = o0 + p.out_plane_stride * 2 + (long long)(c0 >> 6) * 128 + (c0 & 63) + j * 8;
      *reinterpret_cast<uint4 *>(o0 + (long long)c0 * 2 + j * 16) = hw;
      *reinterpret_cast<uint2 *>(o1) = qv;
      *reinterpret_cast<uint2 *>(o1 + 64) = qr;
    }
  } else if (F8 && !out_f32 && !(p.flags & CTPN_F_OUT_BF16X2)) {
    // F16F8 planes: fp16 words, then the e4m3 copies of the values and of the residuals (8 + 8 words)
    uint32_t wh[16], wq[16];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      f16f8_quad(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3], p.out_s, p.out_t, p.out_rs, wh[2 * i], wh[2 * i + 1], wq[i], wq[8 + i]);
    }
    const int j = lane & 3;
    const bool st_ok = c0 < p.Cout && !CTPN_DBG(p, 8);
    // plane 0: 64 contiguous bytes per pixel (32 fp16).  plane 1: the pixel's 128-byte block of channel block
    // c0 / 64 holds values at +0 and residuals at +64; this chunk owns 32 bytes of each
    uint8_t *obase = reinterpret_cast<uint8_t *>(p.out);
    store_transposed(stage_w, wh, obase + (long long)c0 * 2 + j * 16, (long long)p.Cout * 2, e, st_ok, small, lane);
    store_transposed(stage_w, wq, obase + p.out_plane_stride * 2 + (long long)(c0 >> 6) * 128 + (c0 & 63) + (j >> 1) * 64 + (j & 1) * 16,
                     (long long)p.Cout * 2, e, st_ok, small, lane);
  } else if (!out_f32) {
    uint32_t w[P][16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      uint32_t t[P];
      split_planes2<P>(v[2 * i], v[2 * i + 1], t);
#pragma unroll
      for (int pl = 0; pl < P; ++pl) w[pl][i] = t[pl];
    }
#pragma unroll
    for (int pl = 0; pl < P; ++pl) {
      uint8_t *obase = reinterpret_cast<uint8_t *>(reinterpret_cast<__nv_bfloat16 *>(p.out) + (long long)pl * p.out_plane_stride + c0 + (lane & 3) * 8);
      store_transposed(stage_w, w[pl], obase, (long long)p.Cout * 2, e, c0 < p.Cout && !CTPN_DBG(p, 8), small, lane);
    }
  } else if (e.ok && c0 < p.Cout && !CTPN_DBG(p, 8)) {
    float4 *dst = reinterpret_cast<float4 *>(reinterpret_cast<float *>(p.out) + e.pix * p.Cout + c0);
#pragma unroll
    for (int q = 0; q < 8; ++q) dst[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  }
}

// MC = 1: launched as 2-CTA clusters.  The two CTAs of a cluster work on two pixel tiles of the SAME output-channel tile in
// lock step; each loads half of every weight (B) tile and TMA-multicasts it into both CTAs' shared memory, which halves the
// L2 -> SM weight traffic.  A weight stage is free when BOTH CTAs' MMAs have read it, so its 'empty' barrier counts the
// arrivals of the two consumer warpgroups of each CTA.
// F8 = 1 (with P = 2 stage slots): the F16F8 arithmetic -- plane 0 holds fp16 operands (fp16 wgmma into the main
// accumulator), plane 1 the K-concatenated e4m3 copies (e4m3 wgmma, K = 32, into the cross accumulator): 4 + 4 tensor
// core instructions per (tap, channel block) where two bf16 planes need 12.
// PR = 1 (CTPN_F_PROMOTE, P = 3 only): the main accumulator is restarted at every pipeline step (one tap of one channel
// block, K = 64) and each step's partial sum is added into a third register array with round-to-nearest float32 adds, so
// the tensor core's truncating adds run over chains of 4 MMAs instead of 4 * 9 * Cin / 64.  Each step commits its main and
// its cross MMAs as two groups; the promotion waits for the main group only and overlaps the cross MMAs.
// Epilogue handoff (PR = 0): the MMA warpgroups write a 64-channel half of the combined tile into the staging buffer and
// arrive on epiF (256 arrivals); the epilogue warpgroup lifts its pixel's 64 channels into registers and arrives on epiE
// (128 arrivals) before it converts and stores them, so the MMA warpgroups wait for one shared-memory pass per half.
template <int BN, int P, int TAPS, int MC, int F8, int PR = 0>
__global__ void __launch_bounds__(kTcThreads<BN, PR>, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const ConvTcParams p) {
  using namespace ptx;
  constexpr int kBBytes = BN * 128;
  constexpr bool EW = kEpiWarpgroup<BN, PR>;
  static_assert(!F8 || P == 2, "F16F8 uses two stage slots per operand");
  static_assert(!PR || (P == 3 && !F8), "promotion is built for three bf16 planes");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t ring_a = (raw + 1023u) & ~1023u;
  const uint32_t a_stage = (uint32_t)P * p.patch_bytes, b_stage = (uint32_t)P * kBBytes;
  const uint32_t ring_b = ring_a + (uint32_t)p.stages_a * a_stage;
  float *epi = reinterpret_cast<float *>(smem_raw + (ring_b - raw) + (size_t)p.stages_b * b_stage);
  uint4 *xpose = reinterpret_cast<uint4 *>(reinterpret_cast<uint8_t *>(epi) + kEpiBytes);   // EW: the transpose blocks
  uint8_t *ctrl = reinterpret_cast<uint8_t *>(epi) + kEpiBytes + (EW ? kXposeBytes : 0);
  const uint32_t fullA = smem_u32(ctrl), emptyA = fullA + 8 * kMaxStages;
  const uint32_t fullB = emptyA + 8 * kMaxStages, emptyB = fullB + 8 * kMaxStages;
  const uint32_t epiF = emptyB + 8 * kMaxStages, epiE = epiF + 8;

  // warp index through a shuffle so the compiler knows it is warp-uniform: the role loops below are executed by
  // whole warps with uniform control flow and only the instruction issue is predicated on one elected lane --
  // otherwise every TMA instruction gets wrapped in a per-lane 'waterfall' loop.
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    for (int s = 0; s < kMaxStages; ++s) {
      mbar_init(fullA + 8 * s, 1);
      mbar_init(emptyA + 8 * s, 2);             // the two consumer warpgroups
      mbar_init(fullB + 8 * s, 1);
      mbar_init(emptyB + 8 * s, MC ? 4 : 2);    // ... of each CTA of the cluster
    }
    mbar_init(epiF, 256);
    mbar_init(epiE, 128);
    fence_mbar_init();
  }
  __syncthreads();
  if (MC) cluster_sync_all();      // the peer's barriers are initialised before anything is multicast into them
  const uint32_t rank = MC ? cluster_ctarank() : 0u;
  // persistent loop over work units: a tile, or (MC) a pair of pixel tiles x one channel tile shared by the cluster
  const int u_begin = MC ? (int)(blockIdx.x >> 1) : (int)blockIdx.x, u_step = MC ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  auto unit_tile = [&](int u, int &mt, int &nt) {
    nt = u % p.tiles_n;
    mt = u / p.tiles_n;
    if (MC) mt = min(2 * mt + (int)rank, p.m_tiles - 1);   // odd tile count: the last pair computes the same tile twice
  };

  const int kblocks = p.Cin / 64;
  const int tiles_per_img = p.tiles_x * p.tiles_y;
  constexpr int halo = TAPS == 9 ? 1 : 0;

  // registers (EW): 128 x 24 + 256 x 168 + 128 x 152 = the 65 536 of the SM
  if (warp < 4) {
    if (EW) regs_dealloc<24>();
    else regs_dealloc<40>();
    if (warp == 1) {
      // ===== activation (A) producer: one halo patch per plane per channel block =====
      int s = 0;
      uint32_t ph = 0;
      for (int u = u_begin; u < p.total_units; u += u_step) {
        int mt, nt;
        unit_tile(u, mt, nt);
        const int b = mt / tiles_per_img, r = mt % tiles_per_img;
        const int y0 = (r / p.tiles_x) * p.TH - halo, x0 = (r % p.tiles_x) * p.TW - halo;
        for (int kb = 0; kb < kblocks; ++kb) {
          mbar_wait(emptyA + 8 * s, ph ^ 1u);
          if (elect_one()) {
            if (CTPN_DBG(p, 2)) { mbar_arrive(fullA + 8 * s); }
            else {
              mbar_arrive_expect_tx(fullA + 8 * s, (uint32_t)P * (uint32_t)p.patch_tx_bytes);
              for (int pl = 0; pl < P; ++pl)
                tma_load_4d(&tmap_a, fullA + 8 * s, ring_a + s * a_stage + pl * p.patch_bytes, kb * 64, x0, y0, pl * p.B + b);
            }
          }
          __syncwarp();
          if (++s == p.stages_a) { s = 0; ph ^= 1u; }
        }
      }
    } else if (warp == 0) {
      // ===== weight (B) producer: one [BN][64] tile per plane per (channel block, tap) =====
      int s = 0;
      uint32_t ph = 0;
      for (int u = u_begin; u < p.total_units; u += u_step) {
        int mt, nt;
        unit_tile(u, mt, nt);
        for (int kb = 0; kb < kblocks; ++kb) {
          for (int tap = 0; tap < TAPS; ++tap) {
            mbar_wait(emptyB + 8 * s, ph ^ 1u);
            if (elect_one()) {
              if (CTPN_DBG(p, 1)) { mbar_arrive(fullB + 8 * s); }
              else {
                mbar_arrive_expect_tx(fullB + 8 * s, b_stage);   // MC: own half + the peer's multicast half
                for (int pl = 0; pl < P; ++pl) {
                  if (MC)
                    tma_load_2d_mc(&tmap_b, fullB + 8 * s, ring_b + s * b_stage + pl * kBBytes + rank * (kBBytes / 2),
                                   tap * p.Cin + kb * 64, pl * p.cout_pad + nt * BN + (int)rank * (BN / 2), (uint16_t)3);
                  else
                    tma_load_2d(&tmap_b, fullB + 8 * s, ring_b + s * b_stage + pl * kBBytes, tap * p.Cin + kb * 64,
                                pl * p.cout_pad + nt * BN);
                }
              }
            }
            __syncwarp();
            if (++s == p.stages_b) { s = 0; ph ^= 1u; }
          }
        }
      }
    }
  } else if (EW && warp >= 12) {
    regs_alloc<152>();
    // ===== epilogue warpgroup: thread = pixel m of the tile; per 64-channel half, lift the pixel's two 32-channel chunks
    // from the staging buffer, free the buffer, then convert and store them =====
    const int m = (warp & 3) * 32 + lane;
    uint4 *stage_w = xpose + (warp & 3) * 32;
    uint32_t eph = 0;
    if (!CTPN_DBG(p, 16)) {
      for (int u = u_begin; u < p.total_units; u += u_step) {
        int mt, nt;
        unit_tile(u, mt, nt);
        EpiPixel e;
        epi_pixel(p, mt, m, lane, e);
#pragma unroll 1
        for (int c2 = 0; c2 < BN / 64; ++c2) {
          float v[2][32];
          mbar_wait(epiF, eph);
#pragma unroll
          for (int es = 0; es < 2; ++es) {
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              const float4 t = *reinterpret_cast<const float4 *>(epi + es * 4096 + m * 32 + ((q ^ (m & 7)) << 2));
              v[es][4 * q + 0] = t.x; v[es][4 * q + 1] = t.y; v[es][4 * q + 2] = t.z; v[es][4 * q + 3] = t.w;
            }
          }
          mbar_arrive(epiE);
          eph ^= 1u;
#pragma unroll
          for (int es = 0; es < 2; ++es) epi_chunk<P, F8>(p, e, v[es], nt * BN + (2 * c2 + es) * 32, stage_w, true, false, lane);
        }
      }
    }
  } else {
    if (EW) regs_alloc<168>();
    else regs_alloc<232>();
    // ===== MMA warpgroups: warpgroup wg multiplies tile rows [64 wg, 64 wg + 64) (pixel tile rows 8 wg .. 8 wg + 7) against
    // all BN channels, then hands the tile to the epilogue warpgroup (PR: runs the epilogue itself) =====
    const int wg = (warp >> 2) - 1;
    const bool leader = (threadIdx.x & 127) == 0;
    constexpr int R = BN / 2;                  // accumulator registers per thread (64 x BN per warpgroup)
    float accm[R], accc[R];                    // main and (P > 1) cross accumulators
    float accs[R];                             // PR: round-to-nearest sum of the promoted main chains (unused otherwise)
#ifdef CTPN_DEBUG
    const int pe = PR ? p.promote_every : 1;   // steps per main chain
#else
    constexpr int pe = 1;
#endif
    // Descriptors are (per-stage low word) + compile-time offsets: planes, taps and k-slices are fully unrolled.
    constexpr uint32_t kPatch16 = (TAPS == 9 ? 23552u : 16384u) >> 4;   // plane stride of the A stage, in 16-B units
    constexpr uint32_t kB16 = (uint32_t)kBBytes >> 4;
    constexpr uint32_t kHiB = gmma_desc_hi(1024);
    const uint32_t hi_a = gmma_desc_hi((uint32_t)p.group_stride_bytes);
    const uint32_t wg_off = (uint32_t)wg * 8u * (uint32_t)p.group_stride_bytes;   // 8 row groups of 8 pixels per warpgroup
    int sa = 0, sb = 0, prev_b = -1, prev_a = -1;
    uint32_t pha = 0, phb = 0, eph = 0;
    // accumulator fragments -> staging: 64 channels (fragments 8 c2 .. 8 c2 + 7) as two [128 pixels][32 channels] float32
    // chunks, 16-byte pieces XOR-swizzled by pixel & 7
    const int frow = wg * 64 + (warp & 3) * 16 + (lane >> 2);     // accumulator fragment rows frow, frow + 8
    auto stage_half = [&](int c2) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int i8 = c2 * 8 + j, q = 2 * (j & 3) + ((lane & 3) >> 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = frow + 8 * h;
          *reinterpret_cast<float2 *>(epi + (j >> 2) * 4096 + row * 32 + ((q ^ (row & 7)) << 2) + 2 * (lane & 1)) =
              make_float2(accm[4 * i8 + 2 * h], accm[4 * i8 + 2 * h + 1]);
        }
      }
    };
    // a weight stage (and after its last tap an activation stage) is released once the MMAs that read it have completed
    auto release = [&](int sbx, int sax) {
      if (leader) {
        if (MC) {
          mbar_arrive_cluster(emptyB + 8 * sbx, 0u);
          mbar_arrive_cluster(emptyB + 8 * sbx, 1u);
        } else {
          mbar_arrive(emptyB + 8 * sbx);
        }
        if (sax >= 0) mbar_arrive(emptyA + 8 * sax);
      }
    };
    for (int u = u_begin; u < p.total_units; u += u_step) {
      if (PR) {
#pragma unroll
        for (int i = 0; i < R; ++i) accs[i] = 0.f;
      }
      for (int kb = 0; kb < kblocks; ++kb) {
        if (p.stages_a == 1 && prev_a >= 0) {   // a single activation stage: it must be free before its next load
          wgmma_wait<0>();
          release(prev_b, prev_a);
          prev_b = prev_a = -1;
        }
        mbar_wait(fullA + 8 * sa, pha);
        const uint32_t a_lo = gmma_desc_lo(ring_a + sa * a_stage + wg_off);
#pragma unroll
        for (int tap = 0; tap < TAPS; ++tap) {
          mbar_wait(fullB + 8 * sb, phb);
          const uint32_t b_lo = gmma_desc_lo(ring_b + sb * b_stage);
          constexpr int kPW = 10;
          const uint32_t view16 = TAPS == 9 ? (uint32_t)((tap / 3) * kPW + tap % 3) * 8u : 0u;
          const uint32_t not_first = (kb | tap) != 0;
          const int step = kb * TAPS + tap;
          wgmma_fence();
          if (!CTPN_DBG(p, 4)) {
            if (F8) {
#pragma unroll
              for (int k = 0; k < 4; ++k)     // fp16 x fp16, K = 16 (32 B) per instruction
                wgmma_f16(accm, ((uint64_t)hi_a << 32) | (a_lo + view16 + 2u * k), ((uint64_t)kHiB << 32) | (b_lo + 2u * k),
                          k == 0 ? not_first : 1u);
#pragma unroll
              for (int k = 0; k < 4; ++k)     // e4m3 x e4m3, K = 32 (32 B): k 0,1 = value x residual, k 2,3 = residual x value
                wgmma_e4m3(accc, ((uint64_t)hi_a << 32) | (a_lo + kPatch16 + view16 + 2u * k),
                           ((uint64_t)kHiB << 32) | (b_lo + kB16 + 2u * k), k == 0 ? not_first : 1u);
            } else if (PR) {
              const uint32_t chain_on = step % pe != 0;     // 0: this step starts a new main chain
#pragma unroll
              for (int k = 0; k < 4; ++k)
                wgmma_bf16(accm, ((uint64_t)hi_a << 32) | (a_lo + view16 + 2u * k), ((uint64_t)kHiB << 32) | (b_lo + 2u * k),
                           k == 0 ? chain_on : 1u);
              wgmma_commit();                               // the main group: the promotion below waits for it alone
#pragma unroll
              for (int i = 0; i < P; ++i) {
#pragma unroll
                for (int j = (i == 0); j < P - i; ++j) {
#pragma unroll
                  for (int k = 0; k < 4; ++k) {
                    const uint64_t da = ((uint64_t)hi_a << 32) | (a_lo + i * kPatch16 + view16 + 2u * k);
                    const uint64_t db = ((uint64_t)kHiB << 32) | (b_lo + j * kB16 + 2u * k);
                    wgmma_bf16(accc, da, db, (k == 0 && i == 0 && j == 1) ? not_first : 1u);
                  }
                }
              }
            } else {
#pragma unroll
              for (int i = 0; i < P; ++i) {
#pragma unroll
                for (int j = 0; j < P - i; ++j) {
#pragma unroll
                  for (int k = 0; k < 4; ++k) {   // 64 / K(16); +32 B == +2 in the >>4 address field
                    const uint64_t da = ((uint64_t)hi_a << 32) | (a_lo + i * kPatch16 + view16 + 2u * k);
                    const uint64_t db = ((uint64_t)kHiB << 32) | (b_lo + j * kB16 + 2u * k);
                    if (i + j == 0) wgmma_bf16(accm, da, db, k == 0 ? not_first : 1u);
                    else wgmma_bf16(accc, da, db, (k == 0 && i == 0 && j == 1) ? not_first : 1u);
                  }
                }
              }
            }
          }
          wgmma_commit();
          // the previous step's MMAs are done: free its stages (PR: groups retire in order, so this step's main group is done too)
          wgmma_wait<1>();
          if (prev_b >= 0) release(prev_b, prev_a);
          prev_b = sb;
          prev_a = tap == TAPS - 1 ? sa : -1;
          if (PR && ((step + 1) % pe == 0 || step == kblocks * TAPS - 1)) {
            wgmma_fence_regs(accm);
#pragma unroll
            for (int i = 0; i < R; ++i) accs[i] = __fadd_rn(accs[i], accm[i]);   // (0 + x is exact)
          }
          if (++sb == p.stages_b) { sb = 0; phb ^= 1u; }
        }
        if (++sa == p.stages_a) { sa = 0; pha ^= 1u; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(accm);
      if (P > 1) wgmma_fence_regs(accc);
      if (prev_b >= 0) release(prev_b, prev_a);
      prev_b = prev_a = -1;
      // main (+ cross): kept apart during the K loop because the tensor core truncates when it adds into float32
      if (P > 1) {
#pragma unroll
        for (int i = 0; i < R; ++i)
          accm[i] = F8 ? __fmaf_rn(accc[i], p.inv_cross, accm[i] * p.inv_main) : PR ? __fadd_rn(accs[i], accc[i]) : accm[i] + accc[i];
      }

      if (CTPN_DBG(p, 16)) continue;
      if (EW) {
        // +bias -> ReLU here, where the thread's 2 x BN / 8 channels come with few loads, then hand the tile over in
        // 64-channel halves; the epilogue warpgroup frees the buffer once it has read a half
        const float *bt = p.bias + (u % p.tiles_n) * BN + 2 * (lane & 3);   // accm[4 i8 + 2 h + k]: channel 8 i8 + 2 (lane & 3) + k
#pragma unroll
        for (int i8 = 0; i8 < BN / 8; ++i8) {
          const float2 bq = __ldg(reinterpret_cast<const float2 *>(bt + 8 * i8));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            accm[4 * i8 + 2 * h] += bq.x;
            accm[4 * i8 + 2 * h + 1] += bq.y;
          }
        }
        if (p.flags & CTPN_F_RELU) {
#pragma unroll
          for (int i = 0; i < R; ++i) accm[i] = fmaxf(accm[i], 0.f);
        }
#pragma unroll
        for (int c2 = 0; c2 < BN / 64; ++c2) {
          mbar_wait(epiE, eph ^ 1u);
          stage_half(c2);
          mbar_arrive(epiF);
          eph ^= 1u;
        }
      } else {
        // both MMA warpgroups run the epilogue: warp cw = set (even / odd 32-channel chunks) x quarter of the 128 pixels
        const int cw = warp - 4, eset = cw >> 2, quarter = cw & 3;
        const int m = quarter * 32 + lane;
        int mt, nt;
        unit_tile(u, mt, nt);
        EpiPixel e;
        epi_pixel(p, mt, m, lane, e);
        // the 32 staging rows a warp reads back are its own, and once read they serve as its store-transpose block
        uint4 *stage_w = reinterpret_cast<uint4 *>(epi + eset * 4096 + quarter * 1024);
#pragma unroll
        for (int c2 = 0; c2 < BN / 64; ++c2) {
          named_sync(1, 256);           // the previous chunk pair has been read
          stage_half(c2);
          named_sync(1, 256);
          float v[32];
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const float4 t = *reinterpret_cast<const float4 *>(epi + eset * 4096 + m * 32 + ((q ^ (m & 7)) << 2));
            v[4 * q + 0] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
          }
          epi_chunk<P, F8>(p, e, v, nt * BN + (2 * c2 + eset) * 32, stage_w, false, true, lane);
        }
      }
    }
  }
  __syncthreads();
  if (MC) cluster_sync_all();      // no CTA leaves while its peer can still signal its barriers
}


// ---- host side -------------------------------------------------------------------------------
// Per-device launch state: SM count, the dynamic-shared-memory attribute and the co-resident cluster count of every
// kernel instantiation (set once per device, under a mutex), and a small cache of encoded tensor maps keyed by the
// tensor they describe, so that a steady-state ctpn_conv3x3 call does no driver work besides the launch itself.
constexpr int kMaxDevices = 64;
static std::mutex g_mu;
static int g_sms[kMaxDevices];

struct Tuning { int debug = 0, bn = 0, stages_a = 0, stages_b = 0, mcast = 1, promote = 1; };
static const Tuning &tuning() {            // read once at first use; overrides exist only in the test library
  static const Tuning t = [] {
    Tuning v;
#ifdef CTPN_DEBUG
    auto env_int = [](const char *name, int dflt) { const char *e = getenv(name); return e ? atoi(e) : dflt; };
    v.debug = env_int("CTPN_TC_DEBUG", 0);
    v.bn = env_int("CTPN_TC_BN", 0);
    v.stages_a = env_int("CTPN_TC_STAGES_A", 0);
    v.stages_b = env_int("CTPN_TC_STAGES_B", 0);
    v.mcast = env_int("CTPN_TC_MCAST", 1);
    v.promote = std::max(1, env_int("CTPN_TC_PROMOTE", 1));   // CTPN_F_PROMOTE: pipeline steps per promoted main chain
#endif
    return v;
  }();
  return t;
}

struct TmapKey {
  const void *ptr;
  unsigned long long d0, d1, d2, d3;
  unsigned b0, b1, b2, b3;
  int dev;
  bool operator==(const TmapKey &o) const {
    return ptr == o.ptr && d0 == o.d0 && d1 == o.d1 && d2 == o.d2 && d3 == o.d3 && b0 == o.b0 && b1 == o.b1 && b2 == o.b2 &&
           b3 == o.b3 && dev == o.dev;
  }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey &k) const {
    size_t h = std::hash<const void *>()(k.ptr);
    for (unsigned long long v : {k.d0, k.d1, k.d2, k.d3, (unsigned long long)k.b0, (unsigned long long)k.b1,
                                 (unsigned long long)k.b2, (unsigned long long)k.b3, (unsigned long long)k.dev})
      h = h * 1000003u ^ std::hash<unsigned long long>()(v);
    return h;
  }
};
static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmaps;

// bf16 tensor map (128-B swizzle) of `rank` dimensions, from the cache or freshly encoded
static int cached_tmap(int dev, CUtensorMap *out, const void *ptr, int rank, const cuuint64_t *dims, const cuuint64_t *strides,
                       const cuuint32_t *box) {
  TmapKey k{ptr, dims[0], dims[1], rank > 2 ? dims[2] : 0, rank > 3 ? dims[3] : 0, box[0], box[1], rank > 2 ? box[2] : 0,
            rank > 3 ? box[3] : 0, dev};
  std::lock_guard<std::mutex> lock(g_mu);
  auto it = g_tmaps.find(k);
  if (it != g_tmaps.end()) { *out = it->second; return CTPN_OK; }
  EncodeTiledFn enc = nullptr;
  int rc = tma_get_encode(&enc);
  if (rc) return rc;
  if ((rc = tma_encode_bf16(enc, out, const_cast<void *>(ptr), rank, dims, strides, box))) return rc;
  if (g_tmaps.size() >= 1024) g_tmaps.clear();      // bounded: callers cycle through a handful of buffers
  g_tmaps.emplace(k, *out);
  return CTPN_OK;
}

template <int BN, int P, int TAPS, int MC, int F8 = 0, int PR = 0>
static int launch_bn(int dev, const CUtensorMap &ta, const CUtensorMap &tb, ConvTcParams &p, cudaStream_t st) {
  const size_t a_stage = (size_t)p.planes * p.patch_bytes, b_stage = (size_t)p.planes * BN * 128;
  const size_t epi_bytes = kEpiBytes + (kEpiWarpgroup<BN, PR> ? kXposeBytes : 0);     // staging (+ the epilogue warpgroup's transpose blocks)
  const size_t budget = 227 * 1024 - 1024 - kCtrlBytes - epi_bytes;
  // activation ring: two stages when they leave room for at least two weight stages, else one
  int sa = (2 * a_stage + 2 * b_stage <= budget) ? 2 : 1;
  if (p.taps == 1) sa = (int)std::min<size_t>(4, std::max<size_t>(1, (budget / 2) / a_stage));
  // at least two weight stages: the consumers free a stage only after the MMAs of the following one have been issued
  CTPN_REQUIRE(sa * a_stage + 2 * b_stage <= budget, "conv_tc: pipeline stages (%zu + 2 x %zu B) do not fit in shared memory", a_stage, b_stage);
  int sb = (int)((budget - sa * a_stage) / b_stage);
  if (sb > kMaxStages) sb = kMaxStages;
  if (tuning().stages_a > 0) sa = std::max(1, std::min(sa, tuning().stages_a));
  if (tuning().stages_b > 0) sb = std::max(2, std::min(sb, tuning().stages_b));
  p.stages_a = sa;
  p.stages_b = sb;
  const size_t smem = 1024 + sa * a_stage + sb * b_stage + epi_bytes + kCtrlBytes;
  CTPN_REQUIRE(smem <= 227 * 1024, "conv_tc: %zu bytes of shared memory", smem);
  auto kernel = conv_tc_kernel<BN, P, TAPS, MC, F8, PR>;
  static bool attr_set[kMaxDevices];
  static int max_clusters[kMaxDevices];     // co-resident 2-CTA clusters of this instantiation (one CTA per SM)
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = 2; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
  cfg.blockDim = dim3(kTcThreads<BN, PR>);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.attrs = &attr;
  cfg.numAttrs = MC ? 1 : 0;
  {
    std::lock_guard<std::mutex> lock(g_mu);
    if (!attr_set[dev]) {
      CTPN_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));   // the largest layout of any call (stage counts vary per layer)
      if (MC) {
        cfg.gridDim = dim3(2 * (g_sms[dev] / 2));
        int n = 0;
        CTPN_CUDA(cudaOccupancyMaxActiveClusters(&n, kernel, &cfg));
        CTPN_REQUIRE(n > 0, "conv_tc: no 2-CTA cluster of this kernel fits on the device");
        max_clusters[dev] = n;
      }
      attr_set[dev] = true;
    }
  }
  char label[128];
  if (prof_enabled()) snprintf(label, sizeof(label), "conv_tc t%d %dx%dx%d c%d-%d %s%d bn%d%s%s", p.taps, p.B, p.H, p.W, p.Cin, p.Cout, F8 ? "f16f8 p" : "p", p.planes, BN, MC ? " mc" : "", PR ? " promote" : "");
  ProfScope prof(label, p.work, st);
  if (MC) cfg.gridDim = dim3(2 * std::min(max_clusters[dev], p.total_units));
  else cfg.gridDim = dim3(std::min(p.total_units, g_sms[dev]));
  CTPN_CUDA(cudaLaunchKernelEx(&cfg, kernel, ta, tb, p));
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

int conv_tc_run(const void *in_planes, const void *w_planes, const float *bias, void *out, int B, int H, int W, int cin,
                int cout, int taps, int planes, int flags, const QuantScales *q, const int *ext, int ext_shift, void *stream) {
  const bool f8 = q != nullptr, promote = (flags & CTPN_F_PROMOTE) != 0;
  CTPN_REQUIRE(f8 || !(flags & CTPN_F_OUT_BF16X2), "ctpn_conv3x3: CTPN_F_OUT_BF16X2 is a flag of ctpn_conv3x3_f16f8");
  CTPN_REQUIRE(!(promote && f8), "ctpn_conv3x3_f16f8: CTPN_F_PROMOTE is a flag of ctpn_conv3x3 with planes = 3");
  CTPN_REQUIRE(!promote || planes == 3, "ctpn_conv3x3: CTPN_F_PROMOTE needs planes = 3 (got %d)", planes);
  CTPN_REQUIRE(in_planes && w_planes && bias && out, "ctpn_conv3x3: null pointer");
  CTPN_REQUIRE(taps == 9 || taps == 1, "ctpn_conv3x3: taps must be 9 or 1 (got %d)", taps);
  CTPN_REQUIRE(planes >= 1 && planes <= 3, "ctpn_conv3x3: planes must be 1..3 (got %d)", planes);
  CTPN_REQUIRE(cin % 64 == 0 && cin >= 64, "ctpn_conv3x3: Cin must be a multiple of 64 (got %d)", cin);
  CTPN_REQUIRE(cout % 64 == 0 && cout >= 64, "ctpn_conv3x3: Cout must be a multiple of 64 (got %d)", cout);
  CTPN_REQUIRE(B > 0 && H > 0 && W > 0, "ctpn_conv3x3: bad shape");
  const bool pool = flags & CTPN_F_POOL;
  CTPN_REQUIRE(!pool || (taps == 9 && H >= 2 && W >= 2), "ctpn_conv3x3: pooling needs taps=9 and H,W >= 2");
  const bool stack_in = flags & CTPN_F_STACK_IN, stack_out = flags & CTPN_F_STACK_OUT;
  CTPN_REQUIRE(!stack_in || (taps == 9 && !pool), "ctpn_conv3x3: CTPN_F_STACK_IN needs taps=9 and no pooling");
  CTPN_REQUIRE(!stack_out || !(flags & CTPN_F_OUT_F32), "ctpn_conv3x3: stacked output is a plane format");
  const int img_B = B, img_H = H;
  if (stack_in) {          // the kernel sees one image of B * (H + 1) rows
    CTPN_REQUIRE((long long)B * (H + 1) < (1ll << 30), "ctpn_conv3x3: stack too tall");
    H = B * (H + 1);
    B = 1;
  }
  int dev = 0, rc;
  CTPN_CUDA(cudaGetDevice(&dev));
  CTPN_REQUIRE(dev >= 0 && dev < kMaxDevices, "ctpn_conv3x3: device index %d not supported", dev);
  {
    std::lock_guard<std::mutex> lock(g_mu);
    if (g_sms[dev] == 0) CTPN_CUDA(cudaDeviceGetAttribute(&g_sms[dev], cudaDevAttrMultiProcessorCount, dev));
  }

  ConvTcParams p;
  memset(&p, 0, sizeof(p));
  p.B = B; p.H = H; p.W = W; p.Cin = cin; p.Cout = cout; p.taps = taps; p.planes = planes; p.flags = flags;
  if (taps == 9) {   // 16 x 8 pixel tile: one 8-row wgmma group per tile row, halo patch 18 x 10
    p.TH = 16; p.TW = 8; p.tw_log2 = 3;
    p.PW = 10;
    p.group_stride_bytes = p.PW * 128;
    p.patch_tx_bytes = p.PW * 18 * 128;
    p.patch_bytes = (int)align_up((size_t)p.patch_tx_bytes, 1024);
  } else {           // flat 128-pixel tile along W (callers pass matmuls as H = 1)
    p.TH = 1; p.TW = 128; p.tw_log2 = 7;
    p.PW = 128;
    p.group_stride_bytes = 1024;
    p.patch_tx_bytes = 128 * 128;
    p.patch_bytes = 128 * 128;
  }
  p.tiles_x = ceil_div(W, p.TW);
  p.tiles_y = ceil_div(H, p.TH);
  p.Ho = pool ? H / 2 : H;
  p.Wo = pool ? W / 2 : W;
  p.bias = bias;
  p.out = out;
  p.work = 2.0 * img_B * img_H * W * (double)taps * cin * cout;
  p.in_stack_h = stack_in ? img_H + 1 : 0;
  const int img_Ho = pool ? img_H / 2 : img_H;
  p.out_rows = img_Ho + (stack_out ? 1 : 0);
  p.out_stacked = stack_out ? 1 : 0;
  p.out_plane_stride = (long long)img_B * p.out_rows * p.Wo * cout;
  p.cout_pad = cout;
  p.ext = ext;
  p.ext_shift = ext_shift;
  p.ext_n = img_B;
  if (f8) {
    CTPN_REQUIRE(q->inv_main > 0.f && q->inv_cross > 0.f && q->out_s > 0.f && q->out_t > 0.f, "ctpn_conv3x3_f16f8: scales must be positive");
    p.inv_main = q->inv_main; p.inv_cross = q->inv_cross; p.out_s = q->out_s; p.out_t = q->out_t;
    p.out_rs = kResidualGain * q->out_t / q->out_s;
  }
  p.debug = tuning().debug;
  p.promote_every = tuning().promote;

  // N tile: 256 halves the A traffic per MAC; with two accumulators per tile (P > 1) it would need 256 accumulator
  // registers per consumer thread, so those stay at 128.
  int BN = tuning().bn > 0 ? tuning().bn : (planes == 1 ? 256 : 128);
  if (!(BN == 64 || BN == 128 || BN == 256)) BN = 256;
  if (planes > 1 && BN > 128) BN = 128;   // main + cross accumulators: 2 * BN / 2 registers per thread (F16F8 too)
  while (BN > cout || cout % BN) BN >>= 1;
  const long long m_tiles = (long long)B * p.tiles_x * p.tiles_y;
  // Weight-tile multicast over 2-CTA clusters, for 3x3 layers with at least one pair of pixel tiles and, unpromoted, fewer
  // than kMcMaxTilesPerSm output tiles per SM.  At batch scale the single-CTA kernel is about twice as fast: on one H100
  // (400 W limit), batch 32 x 600x900 F16F8, conv1_2 6.5 against 14.0 ms, conv3_2 5.1 against 8.7 ms and conv4_2 4.5
  // against 8.7 ms (tools/time_conv.py with CTPN_TC_MCAST=0).  Promoted layers keep multicast: their single-CTA kernel
  // runs at BN = 64.
  constexpr long long kMcMaxTilesPerSm = 16;
  const bool mc = taps == 9 && tuning().mcast != 0 && m_tiles >= 2 &&
                  (promote || m_tiles * (cout / BN) < kMcMaxTilesPerSm * g_sms[dev]);
  // promoted single-CTA 3x3 layers (a map of one 16 x 8 tile) run at BN = 64: with three accumulators that kernel
  // spills registers at BN = 128, the multicast and taps = 1 ones do not
  if (promote && taps == 9 && !mc && BN > 64) BN = 64;
  p.tiles_n = cout / BN;
  const long long total = m_tiles * p.tiles_n;
  CTPN_REQUIRE(total < (1ll << 31), "ctpn_conv3x3: too many tiles");
  p.total_tiles = (int)total;
  p.m_tiles = (int)m_tiles;
  p.total_units = mc ? (int)((m_tiles + 1) / 2) * p.tiles_n : p.total_tiles;

  CUtensorMap ta, tb;
  {
    const int halo = taps == 9 ? 1 : 0;
    cuuint64_t dims[4] = {(cuuint64_t)cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)planes * B};
    cuuint64_t strides[3] = {(cuuint64_t)cin * 2, (cuuint64_t)W * cin * 2, (cuuint64_t)H * W * cin * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)p.PW, (cuuint32_t)(p.TH + 2 * halo), 1};
    if ((rc = cached_tmap(dev, &ta, in_planes, 4, dims, strides, box))) return rc;
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)taps * cin, (cuuint64_t)planes * cout};
    cuuint64_t strides[1] = {(cuuint64_t)taps * cin * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)(mc ? BN / 2 : BN)};   // multicast: each CTA of the pair loads half the rows
    if ((rc = cached_tmap(dev, &tb, w_planes, 2, dims, strides, box))) return rc;
  }
  cudaStream_t st = (cudaStream_t)stream;
#define CTPN_TC_CASE(BN_, P_, T_) \
  if (BN == BN_ && planes == P_ && taps == T_) return launch_bn<BN_, P_, T_, 0>(dev, ta, tb, p, st)
#define CTPN_TC_CASE_MC(BN_, P_) \
  if (mc && BN == BN_ && planes == P_) return launch_bn<BN_, P_, 9, 1>(dev, ta, tb, p, st)
  if (f8) {
    if (mc && BN == 128) return launch_bn<128, 2, 9, 1, 1>(dev, ta, tb, p, st);
    if (mc && BN == 64) return launch_bn<64, 2, 9, 1, 1>(dev, ta, tb, p, st);
    if (taps == 9 && BN == 128) return launch_bn<128, 2, 9, 0, 1>(dev, ta, tb, p, st);
    if (taps == 9 && BN == 64) return launch_bn<64, 2, 9, 0, 1>(dev, ta, tb, p, st);
    if (taps == 1 && BN == 128) return launch_bn<128, 2, 1, 0, 1>(dev, ta, tb, p, st);
    if (taps == 1 && BN == 64) return launch_bn<64, 2, 1, 0, 1>(dev, ta, tb, p, st);
    set_error("ctpn_conv3x3_f16f8: no kernel for BN=%d taps=%d", BN, taps);
    return CTPN_ERR_INVALID;
  }
  if (promote) {   // planes == 3
    if (mc && BN == 128) return launch_bn<128, 3, 9, 1, 0, 1>(dev, ta, tb, p, st);
    if (mc && BN == 64) return launch_bn<64, 3, 9, 1, 0, 1>(dev, ta, tb, p, st);
    if (taps == 9 && BN == 64) return launch_bn<64, 3, 9, 0, 0, 1>(dev, ta, tb, p, st);
    if (taps == 1 && BN == 128) return launch_bn<128, 3, 1, 0, 0, 1>(dev, ta, tb, p, st);
    if (taps == 1 && BN == 64) return launch_bn<64, 3, 1, 0, 0, 1>(dev, ta, tb, p, st);
    set_error("ctpn_conv3x3: no promoted kernel for BN=%d taps=%d", BN, taps);
    return CTPN_ERR_INVALID;
  }
  CTPN_TC_CASE_MC(256, 1); CTPN_TC_CASE_MC(128, 1); CTPN_TC_CASE_MC(64, 1);
  CTPN_TC_CASE_MC(128, 2); CTPN_TC_CASE_MC(64, 2);
  CTPN_TC_CASE_MC(128, 3); CTPN_TC_CASE_MC(64, 3);
  CTPN_TC_CASE(256, 1, 9); CTPN_TC_CASE(128, 1, 9); CTPN_TC_CASE(64, 1, 9);
  CTPN_TC_CASE(128, 2, 9); CTPN_TC_CASE(64, 2, 9);
  CTPN_TC_CASE(128, 3, 9); CTPN_TC_CASE(64, 3, 9);
  CTPN_TC_CASE(256, 1, 1); CTPN_TC_CASE(128, 1, 1); CTPN_TC_CASE(64, 1, 1);
  CTPN_TC_CASE(128, 2, 1); CTPN_TC_CASE(64, 2, 1);
  CTPN_TC_CASE(128, 3, 1); CTPN_TC_CASE(64, 3, 1);
#undef CTPN_TC_CASE_MC
#undef CTPN_TC_CASE
  set_error("ctpn_conv3x3: no kernel for BN=%d planes=%d taps=%d", BN, planes, taps);
  return CTPN_ERR_INVALID;
}

}  // namespace ctpn

using namespace ctpn;

extern "C" int ctpn_conv3x3(const void *in_planes, const void *w_planes, const float *bias, void *out, int B, int H,
                            int W, int cin, int cout, int taps, int planes, int flags, void *stream) {
  return conv_tc_run(in_planes, w_planes, bias, out, B, H, W, cin, cout, taps, planes, flags, nullptr, nullptr, 0, stream);
}

extern "C" int ctpn_conv3x3_f16f8(const void *in_planes, const void *w_planes, const float *bias, void *out, int B, int H,
                                  int W, int cin, int cout, int taps, int flags, float inv_main, float inv_cross, float out_s,
                                  float out_t, void *stream) {
  const QuantScales q{inv_main, inv_cross, out_s, out_t};
  return conv_tc_run(in_planes, w_planes, bias, out, B, H, W, cin, cout, taps, 2, flags, &q, nullptr, 0, stream);
}
