// Diagnostic probe (not on the product path): which shared-memory rows does a K-major SWIZZLE_128B wgmma
// A-descriptor fetch when its start address is NOT 1024-byte aligned and its 8-row groups are spaced by an
// arbitrary stride?  The answer decides whether the 9 taps of a 3x3 convolution can be served as shifted
// VIEWS of one halo patch in shared memory instead of 9 separate TMA loads.
//
// A [rows][64] bf16 matrix is TMA-loaded (128B swizzle) into 1024-aligned shared memory; B is the 64x64
// identity, so D[m][n] = A_view[m][n]: the output reveals, for every (m, 16-byte chunk), the element the
// tensor core actually read.  One warpgroup, two m64n64k16 passes (view rows 0-63 and 64-127).
#include <cuda.h>

#include "../common.cuh"
#include "../tc_ptx.cuh"
#include "../tma_host.cuh"
#include "ctpn_b200_testing.h"

namespace ctpn {

__global__ void __launch_bounds__(128, 1)
probe_umma_view_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, int rows,
                       int row0, int group_stride_rows, int base_offset_mode, float *__restrict__ out) {
  using namespace ptx;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t sa = (raw + 1023u) & ~1023u;          // A: rows x 128 B
  const uint32_t sb = sa + ((rows * 128 + 1023) & ~1023);   // B: 64 x 128 B
  __shared__ uint64_t bar;
  const uint32_t bar_load = smem_u32(&bar);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    mbar_init(bar_load, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(bar_load, (uint32_t)(rows * 128 + 64 * 128));
    for (int r = 0; r < rows; r += 64) tma_load_2d(&tmap_a, bar_load, sa + r * 128, 0, r);   // box = 64 x 64
    tma_load_2d(&tmap_b, bar_load, sb, 0, 0);
  }
  mbar_wait(bar_load, 0);
  const uint64_t db = ((uint64_t)gmma_desc_hi(1024) << 32) | gmma_desc_lo(sb);
  for (int half = 0; half < 2; ++half) {
    const uint32_t start = sa + (uint32_t)(row0 + half * 8 * group_stride_rows) * 128u;
    uint32_t hi = gmma_desc_hi((uint32_t)group_stride_rows * 128u);
    if (base_offset_mode == 1) hi |= ((start >> 7) & 7u) << 17;     // descriptor bits [49,52)
    const uint64_t da = ((uint64_t)hi << 32) | gmma_desc_lo(start);
    float d[32];
    wgmma_fence();
    for (int k = 0; k < 4; ++k) wgmma_bf16(d, da + 2ull * k, db + 2ull * k, k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(d);
    for (int i = 0; i < 8; ++i)
      for (int h = 0; h < 2; ++h)
        for (int e = 0; e < 2; ++e)
          out[(half * 64 + warp * 16 + (lane >> 2) + 8 * h) * 64 + 8 * i + 2 * (lane & 3) + e] = d[4 * i + 2 * h + e];
  }
}

}  // namespace ctpn

using namespace ctpn;

// a: device bf16 [rows][64] (rows multiple of 64, <= 512); ident: device bf16 [64][64]; out: device float [128][64]
extern "C" int ctpn_probe_umma_view(const void *a, const void *ident, int rows, int row0, int group_stride_rows,
                                    int base_offset_mode, float *out, void *stream) {
  CTPN_REQUIRE(a && ident && out, "ctpn_probe_umma_view: null pointer");
  CTPN_REQUIRE(rows % 64 == 0 && rows >= 64 && rows <= 512, "ctpn_probe_umma_view: rows must be a multiple of 64 in [64, 512]");
  CTPN_REQUIRE(row0 >= 0 && row0 + 15 * group_stride_rows + 8 <= rows, "ctpn_probe_umma_view: view exceeds the matrix");
  EncodeTiledFn enc = nullptr;
  int rc = tma_get_encode(&enc);
  if (rc) return rc;
  CUtensorMap ta, tb;
  cuuint64_t dims_a[2] = {64, (cuuint64_t)rows}, dims_b[2] = {64, 64}, strides[1] = {128};
  cuuint32_t box[2] = {64, 64};
  if ((rc = tma_encode_bf16(enc, &ta, const_cast<void *>(a), 2, dims_a, strides, box))) return rc;
  if ((rc = tma_encode_bf16(enc, &tb, const_cast<void *>(ident), 2, dims_b, strides, box))) return rc;
  const size_t smem = 1024 + (size_t)((rows * 128 + 1023) & ~1023) + 64 * 128;
  CTPN_CUDA(cudaFuncSetAttribute(probe_umma_view_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  probe_umma_view_kernel<<<1, 128, smem, (cudaStream_t)stream>>>(ta, tb, rows, row0, group_stride_rows, base_offset_mode, out);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}
