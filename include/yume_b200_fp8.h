/* yume_b200_fp8.h — C ABI of the FP8 (e4m3) block-GEMM path in libyume_b200.so (conventions as include/yume_b200.h: device
 * pointers, `stream` a cudaStream_t as void*, no allocation, no synchronisation, capture-safe launches, 0 or a negative
 * YB_ERR_* code).
 *
 * Numerics (every entry point below and the torch twins in the test-suite implement exactly this):
 *   Weights, per output channel n (quantised once on the host):  s_w[n] = amax_n / 448,
 *            Wq[n, k] = e4m3(clamp(W[n, k] * (448 / amax_n), +-448)); an all-zero row has s_w = 0 and Wq = 0.
 *   Activations, per row m and group g of 128 consecutive columns ("1x128 groups"), from the fp32 values the producing kernel
 *            holds: amax = max |x| over the group (NaN elements ignored), inv = 448 / amax (IEEE fp32 division),
 *            scale = amax / 448, q = cvt.rn.satfinite.e4m3(x * inv). When 448 / amax is not finite (amax == 0, or amax below
 *            448 / FLT_MAX ~ 1.3e-36) the group is stored as zeros with inv = scale = 0. A NaN element stays NaN.
 *            The torch twin is (x * inv).clamp(-448, 448).to(torch.float8_e4m3fn) with the same inv and scale: bit-identical.
 *   Scale layout: activation scales are f32 [K / 128, lds], group-major, lds >= M, lds % 4 == 0 (one k-group of 128 rows is
 *            512 contiguous bytes).
 *   GEMM:    out[m, n] = epi( s_w[n] * sum_g s_a[g, m] * (sum_{k in g} Aq[m, k] Wq[n, k]) + bias[n] ).
 *            The inner sum of one 128-wide group is four wgmma m64n128k32 e4m3 into a fresh accumulator; the outer sum is an
 *            fp32 register accumulator updated once per group (promotion: the fp8 tensor-core accumulator keeps fewer bits than
 *            fp32, see DESIGN.md §3).
 */
#ifndef YUME_B200_FP8_H_
#define YUME_B200_FP8_H_

#include "yume_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Epilogue of the fp8 GEMM that has no bf16 counterpart: gelu_tanh(acc + bias), then 1x128 quantisation of each output row
 * segment: e4m3 into `out` (row stride ldo bytes) and f32 scales into out_scale [N / 128, ldos] (the A operand of the next GEMM). */
#define YB_EPI_GELU_FP8 8

typedef struct yb_gemm_fp8_args {
  unsigned struct_bytes;    /* sizeof(yb_gemm_fp8_args): guards against a caller compiled against another layout */
  int M, N, K;              /* K % 128 == 0, N % 128 == 0, any M >= 1 */
  const void* A;            /* e4m3 [M, K], row stride lda bytes (% 16 == 0) */
  const void* a_scale;      /* f32 [K / 128, lds] */
  const void* B;            /* e4m3 [N, K] (nn.Linear.weight layout), row stride ldb bytes (% 16 == 0) */
  const void* b_scale;      /* f32 [N] per-channel weight scale s_w */
  const void* bias;         /* f32 [N] or NULL */
  void* out;                /* YB_EPI_BF16: bf16; YB_EPI_F32: f32; YB_EPI_GATE_RES: f32 residual stream updated in place
                               (out += (acc + bias) * gate[tok_idx[m]][n]); YB_EPI_GELU_FP8: e4m3. Row stride ldo elements. */
  void* out_scale;          /* YB_EPI_GELU_FP8: f32 [N / 128, ldos] */
  const void* gate;         /* YB_EPI_GATE_RES: f32 [U, gate_ld] or NULL (gate == 1) */
  const void* tok_idx;      /* YB_EPI_GATE_RES: int32 [M] or NULL (row 0) */
  long long lda, lds, ldb, ldo, ldos, gate_ld;
  int epilogue;             /* YB_EPI_BF16, YB_EPI_F32, YB_EPI_GATE_RES or YB_EPI_GELU_FP8 */
  int block_n;              /* 0 (automatic) or 128 */
} yb_gemm_fp8_args;

/* ---------------------------------------------------------------------------------------------
 * Persistent warp-specialised e4m3 GEMM (one TMA producer warp, two consumer warpgroups of 64 rows): 128 x 128 output tiles,
 * 128-byte-swizzled 128 x 128 e4m3 operand tiles (one swizzle row = one scale group) with the tile's 128 A-scales loaded by
 * TMA in the same stage. Constraints: M, N, K > 0; N % 128 == 0 and K % 128 == 0 (YB_ERR_SHAPE); A, B, out, scales 16-byte
 * aligned; lda, ldb % 16; ldo % 8 (bf16), % 4 (f32), % 16 (e4m3); lds, ldos % 4 and >= M (YB_ERR_ALIGNMENT / YB_ERR_ARG).
 * ------------------------------------------------------------------------------------------- */
int yb_gemm_fp8(const yb_gemm_fp8_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * yb_ln_modulate (include/yume_b200.h) with an e4m3 output: the fp32 row it computes is quantised in 1x128 groups.
 *   out        e4m3 [L, C], row stride ldo bytes (% 16)
 *   out_scale  f32 [C / 128, lds]
 * One warp per row; the fp32 values are those yb_ln_modulate(out_f32 = 1) writes for the same arguments.
 * Constraints: C in {256, 1024, 3072, 5120} (YB_ERR_SHAPE); adaLN (scale/shift) or affine (weight/lnbias), not both.
 * ------------------------------------------------------------------------------------------- */
int yb_ln_modulate_fp8(const void* x, long long ldx, void* out, long long ldo, void* out_scale, long long lds,
                       const void* scale, const void* shift, long long mod_ld, const void* tok_idx, const void* weight,
                       const void* lnbias, int L, int C, float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * bf16 [M, K] (row stride ldx elements, % 8) -> e4m3 [M, K] (row stride ldo bytes, % 16) + f32 scales [K / 128, lds].
 * Quantises the attention output in front of the o and cross-o projections. K % 128 == 0.
 * ------------------------------------------------------------------------------------------- */
int yb_quant_rows_fp8(const void* x, long long ldx, void* out, long long ldo, void* out_scale, long long lds, int M, int K,
                      void* stream);

#ifdef __cplusplus
}
#endif

#endif  // YUME_B200_FP8_H_
