// Weight packing for the tensor-core layers: TF-layout float32 weights [taps][Cin][Cout] (HWIO flattened,
// lib/networks/network.py:160-170) -> bf16 planes [P][Cout_pad][taps][Cin] (K-major rows of the wgmma B operand).
#include "common.cuh"

namespace ctpn {

// ---- weight packing ---------------------------------------------------------------------------
__global__ void pack_weights_kernel(const float *__restrict__ w, int taps, int cin, int cout, int cout_pad,
                                    int planes, __nv_bfloat16 *__restrict__ out) {
  const long long n = (long long)cout_pad * taps * cin;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int ci = (int)(i % cin);
  const int tap = (int)((i / cin) % taps);
  const int co = (int)(i / ((long long)cin * taps));
  float v = co < cout ? w[((long long)tap * cin + ci) * cout + co] : 0.f;
  __nv_bfloat16 pl[3];
  split_planes(v, planes, pl);
  for (int p = 0; p < planes; ++p) out[(long long)p * n + i] = pl[p];
}

// F16F8 weights (see common.cuh): plane 0 = fp16(w * s_w) [Cout_pad][taps][Cin]; plane 1, per (cout, tap, 64-channel
// block), 128 bytes: e4m3(r_w * 2^11 * t_w)[64] | e4m3(w * t_w)[64] -- the residual half FIRST: it meets the value half of
// the activation row (K 0..63) and the value half meets the activation's residual half (K 64..127).
__global__ void pack_weights_f16f8_kernel(const float *__restrict__ w, int taps, int cin, int cout, int cout_pad, float s_w,
                                          float t_w, __half *__restrict__ hi, uint8_t *__restrict__ cross) {
  const long long n = (long long)cout_pad * taps * cin;
  const long long i2 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 2;     // two adjacent input channels
  if (i2 >= n) return;
  const int ci = (int)(i2 % cin);
  const int tap = (int)((i2 / cin) % taps);
  const int co = (int)(i2 / ((long long)cin * taps));
  float v0 = 0.f, v1 = 0.f;
  if (co < cout) {
    v0 = w[((long long)tap * cin + ci) * cout + co];
    v1 = w[((long long)tap * cin + ci + 1) * cout + co];
  }
  float r0, r1;
  const uint32_t pk = f16x2_split(v0 * s_w, v1 * s_w, r0, r1);
  *reinterpret_cast<uint32_t *>(hi + i2) = pk;
  const float rs = kResidualGain * t_w / s_w;
  const uint32_t q = e4m3x4(r0 * rs, r1 * rs, v0 * t_w, v1 * t_w);
  // byte address of channel ci inside the cross plane: (row of 2*Cin bytes per (cout, tap)) + block * 128 + (ci % 64)
  uint8_t *row = cross + ((long long)co * taps + tap) * (2ll * cin) + (ci / 64) * 128 + (ci % 64);
  *reinterpret_cast<uint16_t *>(row) = (uint16_t)(q & 0xffffu);
  *reinterpret_cast<uint16_t *>(row + 64) = (uint16_t)(q >> 16);
}

}  // namespace ctpn

using namespace ctpn;

extern "C" int ctpn_pack_weights_f16f8(const float *w_tf, int taps, int cin, int cout, int cout_pad, float s_w, float t_w,
                                       void *w_planes_out, void *stream) {
  CTPN_REQUIRE(w_tf && w_planes_out, "ctpn_pack_weights_f16f8: null pointer");
  CTPN_REQUIRE(taps > 0 && cin > 0 && cin % 64 == 0 && cout > 0 && cout_pad >= cout, "ctpn_pack_weights_f16f8: bad shape (Cin %% 64 must be 0)");
  CTPN_REQUIRE(s_w > 0.f && t_w > 0.f, "ctpn_pack_weights_f16f8: scales must be positive");
  const long long n = (long long)cout_pad * taps * cin;
  pack_weights_f16f8_kernel<<<(unsigned)((n / 2 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      w_tf, taps, cin, cout, cout_pad, s_w, t_w, reinterpret_cast<__half *>(w_planes_out),
      reinterpret_cast<uint8_t *>(w_planes_out) + n * 2);
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

extern "C" int ctpn_pack_weights(const float *w_tf, int taps, int cin, int cout, int cout_pad, int planes,
                                 void *w_planes_out, void *stream) {
  CTPN_REQUIRE(w_tf && w_planes_out, "ctpn_pack_weights: null pointer");
  CTPN_REQUIRE(taps > 0 && cin > 0 && cout > 0 && cout_pad >= cout, "ctpn_pack_weights: bad shape");
  CTPN_REQUIRE(planes >= 1 && planes <= 3, "ctpn_pack_weights: planes must be 1..3");
  const long long n = (long long)cout_pad * taps * cin;
  pack_weights_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      w_tf, taps, cin, cout, cout_pad, planes, reinterpret_cast<__nv_bfloat16 *>(w_planes_out));
  CTPN_LAUNCH_CHECK();
  return CTPN_OK;
}

