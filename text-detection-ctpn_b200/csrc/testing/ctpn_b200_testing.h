/*
 * Test-only entry points of libctpn_b200_dbg.so (tests/_native/): float32 SIMT reference kernels with the product
 * kernels' contracts, and a hardware probe.  None of this is in the product library libctpn_b200.so or in
 * include/ctpn_b200.h.  The debug library is the product sources compiled with -DCTPN_DEBUG (ablation switches
 * CTPN_TC_DEBUG / CTPN_C1_DEBUG, tuning overrides CTPN_TC_BN / CTPN_TC_STAGES_* / CTPN_TC_MCAST / CTPN_TC_PROMOTE, the "conv_simt"
 * option of ctpn_net_set_option, which runs every convolution and matmul of a bf16-plane net on the SIMT kernels below and is
 * refused on an F16F8 net) plus the two files in this directory.
 */
#ifndef CTPN_B200_TESTING_H_
#define CTPN_B200_TESTING_H_

#include "../../../include/ctpn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* conv1_1: uint8 BGR image [B][H][W][3] (or float32 blob when src_is_f32) -> 64-channel planes,
 * float32 direct convolution (SIMT reference of ctpn_conv1_1_tc); fuses the mean subtraction of lib/fast_rcnn/test.py:9
 * (lut[256][3] = float32(double(v) - PIXEL_MEANS[c])), bias and ReLU. */
int ctpn_conv1_1(const void *src, int src_is_f32, const float *lut, const float *w_hwio,
                 const float *bias, void *out_planes, int B, int H, int W, int planes, void *stream);


/* Same contract, float32 SIMT implementation (no tensor cores): kernel-level reference used
 * by the tests.  CTPN_F_PROMOTE is accepted and has no effect: these sums already round to nearest. */
int ctpn_conv3x3_simt(const void *in_planes, const void *w_planes, const float *bias, void *out,
                      int B, int H, int W, int cin, int cout, int taps, int planes, int flags,
                      void *stream);

/* The activation scales a calibrated F16F8 net (CTPN_ARITH_F16F8) derived for the outputs of conv1_1 .. conv5_3: s[13],
 * t[13] and the calibration maximum amax[13] from which they were derived (net.cu::calibrate_f16f8).  CTPN_ERR_INVALID
 * before the first forward or on another arithmetic. */
int ctpn_net_f16f8_scales(const ctpn_net_t *net, float *s, float *t, float *amax);


/* ---- hardware probes ---------------------------------------------------------------------
 * Hardware probe used by tests/probe_umma_view.py: reads a [rows][64] bf16 matrix through a wgmma
 * K-major SWIZZLE_128B descriptor that starts at row `row0` with `group_stride_rows` between 8-row
 * groups, against the identity, and returns the 128x64 values the tensor core fetched. */
int ctpn_probe_umma_view(const void *a_bf16, const void *identity_bf16, int rows, int row0,
                         int group_stride_rows, int base_offset_mode, float *out, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CTPN_B200_TESTING_H_ */
