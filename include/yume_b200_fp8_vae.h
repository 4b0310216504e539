/* yume_b200_fp8_vae.h — C ABI of the FP8 (e4m3) path of the Wan2.2 VAE decode convs in libyume_b200.so (conventions as
 * include/yume_b200.h: device pointers, `stream` a cudaStream_t as void*, no allocation, no synchronisation, capture-safe
 * launches, 0 or a negative YB_ERR_* code).
 *
 * Numerics (the quantisers are those of include/yume_b200_fp8.h; the torch twins are oracle/fp8.py):
 *   Weights, per output channel co over all taps x Cp (quantised once on the host): s_w[co] = amax / 448,
 *            Wq[co, tap * Cp + c] = e4m3(W * (448 / amax)); an all-zero row has s_w = 0 and Wq = 0.
 *   Activations, per voxel and group g of 128 consecutive channels: exactly `quantize_act` of the bf16 values yb_vae_rms_act
 *            writes for the same arguments (the value is rounded to bf16 first, then quantised with inv = 448 / amax).
 *   Activation layout: e4m3 [T, H, W, Cp] channels-last, scales f32 [T, Cp / 128, H, W] frame-major (a frame of both is one
 *            contiguous block, so a carried history frame is one copy of each).
 *   Conv:    out[v, co] = epi( s_w[co] * sum_(tap, g) s_a[v + tap, g] * (sum_(c in g) Aq[v + tap, c] Wq[co, tap, c]) + bias[co] ).
 *            v + tap is the tap-shifted input voxel; one outside the input (the causal zero padding in front in time, the zero
 *            padding around in space) has zero data and a zero scale. Each inner sum is four wgmma m64n128k32 e4m3 into a fresh
 *            accumulator, promoted into an fp32 register accumulator with the scale of the tap-shifted voxel (DESIGN.md §3).
 *            Taps are summed in (tap, g) order whatever the tile shape, so every chunking of a stream gives the same bits.
 */
#ifndef YUME_B200_FP8_VAE_H_
#define YUME_B200_FP8_VAE_H_

#include "yume_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct yb_conv3d_fp8_args {
  unsigned struct_bytes;    /* sizeof(yb_conv3d_fp8_args): guards against a caller compiled against another layout */
  const void* x;            /* e4m3 [t_hist + T, H, W, Cp], dense */
  const void* x_scale;      /* f32 [t_hist + T, Cp / 128, H, W], dense */
  const void* w;            /* e4m3 [Cout, kt * kh * kw * Cp] (tap-major, then channel), dense */
  const void* w_scale;      /* f32 [Cout] */
  const void* bias;         /* f32 [Cout] or NULL */
  void* out;                /* bf16 [T * H * W, ldo]: row (t * H + h) * W + w */
  const void* res;          /* YB_EPI_RES_BF16: bf16 residual indexed like out (row stride res_ld), added before the bf16 store */
  long long ldo, res_ld;
  int T, H, W, Cp, Cout;    /* Cp % 128 == 0, Cout % 128 == 0 */
  int kt, kh, kw;           /* (3, 3, 3) or (1, 3, 3) */
  int t_hist;               /* 0: one pass (causal zero padding in front); kt - 1: that many carried frames in front of x */
  int epilogue;             /* YB_EPI_BF16 or YB_EPI_RES_BF16 */
} yb_conv3d_fp8_args;

/* ---------------------------------------------------------------------------------------------
 * Causal 3-D conv with e4m3 operands, unit stride, zero padding by TMA out-of-bounds fill (the zero-padded form of
 * yb_conv3d_causal). Persistent warp-specialised kernel: 128-voxel x 128-channel output tiles, the voxel box TT x TH x TW that
 * yb_conv3d_plan picks for the output extents without kw fusion; per (tap, 128-channel group) one 4-D TMA box of A, one
 * 128 x 128 weight tile and the box's 128 tap-shifted activation scales.
 * Constraints: Cp, Cout % 128 (YB_ERR_SHAPE); taps (3,3,3) or (1,3,3) (YB_ERR_SHAPE); t_hist 0 or kt - 1 (YB_ERR_ARG);
 * (t_hist + T) * H * W * Cp / 128 < 2^31 (YB_ERR_SHAPE); x, w, out 16-byte aligned, ldo % 8, res_ld % 2 (YB_ERR_ALIGNMENT).
 * ------------------------------------------------------------------------------------------- */
int yb_conv3d_fp8(const yb_conv3d_fp8_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * yb_vae_rms_act (include/yume_b200.h) with an e4m3 output: [RMS_norm over channels * gamma] -> [SiLU] -> nearest 2x upsample,
 * each value rounded to bf16 as yb_vae_rms_act stores it, then quantised per voxel and 128-channel group.
 *   out        e4m3 [T, Hs * up, Ws * up, Cp] (dense; channels [C, Cp) are zero)
 *   out_scale  f32 [T, Cp / 128, Hs * up, Ws * up] (dense)
 * Constraints: those of yb_vae_rms_act, and Cp == rup(C, 128) (YB_ERR_SHAPE); out 16-byte aligned, out_scale 4-byte aligned
 * (YB_ERR_ALIGNMENT); out_scale non-NULL (YB_ERR_ARG).
 * ------------------------------------------------------------------------------------------- */
int yb_vae_rms_act_fp8(const void* x, long long ldx, void* out, void* out_scale, const void* gamma, int T, int Hs, int Ws,
                       int C, int Cp, int up, int silu, void* stream);

#ifdef __cplusplus
}
#endif

#endif  // YUME_B200_FP8_VAE_H_
