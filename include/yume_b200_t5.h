/* yume_b200_t5.h — C ABI of the umT5 text-encoder kernels in libyume_b200.so (conventions as include/yume_b200.h: device
 * pointers, `stream` a cudaStream_t as void*, no allocation, no synchronisation, capture-safe launches, 0 or a negative
 * YB_ERR_* code).
 *
 * The encoder's projections run on yb_gemm_bf16 (include/yume_b200.h); this header adds the three steps of a T5 block that the
 * DiT kernels do not cover (wan/modules/t5.py:53-141).
 */
#ifndef YUME_B200_T5_H_
#define YUME_B200_T5_H_

#include "yume_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------------
 * T5 self-attention with a relative-position bias and a key padding mask (T5Attention.forward, wan/modules/t5.py:86-120):
 * no 1/sqrt(d) scale, head_dim 64, non-causal.
 *   q, k, v   bf16 [B*L, heads*64], row strides ldq / ldk / ldv (column slices of the fused q|k|v buffer); sample b owns rows
 *             b*L .. b*L + L - 1, head h columns h*64 .. h*64 + 63
 *   out       bf16 [B*L, heads*64], row stride ldo
 *   bias      f32 [heads, 2L - 1]: the bias of query i and key j is bias[h, j - i + L - 1]
 *   key_mask  uint8 [B, L] (nonzero = attend) or NULL (every key attends)
 * Per (b, h, query i): S_j = q_i . k_j + bias (fp32 accumulation); keys with key_mask == 0 are dropped (the reference's
 * masked_fill with finfo.min gives them exactly zero weight); softmax in fp32 over the kept keys, P rounded to bf16, O = P.V
 * accumulated in fp32, divided by the fp32 normaliser and rounded to bf16. A row with no kept key is written as 0 (callers
 * reject such masks). Any L >= 1: K/V tiles of 64 keys are streamed with an online softmax.
 * Constraints: B, L, heads > 0; ld* >= heads*64 and % 8 == 0; q, k, v, out 16-byte aligned (YB_ERR_ALIGNMENT).
 * ------------------------------------------------------------------------------------------- */
int yb_t5_attention(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* out,
                    long long ldo, int B, int L, int heads, const void* bias, const void* key_mask, void* stream);

/* ---------------------------------------------------------------------------------------------
 * T5LayerNorm (wan/modules/t5.py:53-66): out = x * rsqrt(mean(x^2) + eps) * weight, no mean subtracted, no bias.
 *   x       f32 [L, C] (the residual stream), row stride ldx
 *   out     bf16 (out_f32 = 0) or f32 (out_f32 = 1) [L, C], row stride ldo
 *   weight  f32 [C]
 * fp32 arithmetic, one rounding to the output type. One warp per row, the row held in registers.
 * Constraints: C in {128, 256, 512, 768, 1024, 2048, 4096} (else YB_ERR_SHAPE); x, out, weight 16-byte aligned.
 * ------------------------------------------------------------------------------------------- */
int yb_t5_rmsnorm(const void* x, long long ldx, void* out, long long ldo, int out_f32, const void* weight, int L, int C,
                  float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Gated GELU of T5FeedForward (wan/modules/t5.py:136-138): out = fc1(x) * gelu_tanh(gate(x)).
 *   ug   bf16 [L, 2F], row stride ld_ug: columns 0 .. F-1 are fc1(x) (u), columns F .. 2F-1 are gate(x) (g)
 *   out  bf16 [L, F], row stride ldo
 * out = bf16(u * 0.5 g (1 + tanh(sqrt(2/pi) (g + 0.044715 g^3)))) in fp32 with the accurate tanhf, one rounding.
 * Constraints: F % 8 == 0; ld_ug, ldo % 8 == 0; ug, out 16-byte aligned.
 * ------------------------------------------------------------------------------------------- */
int yb_t5_geglu(const void* ug, long long ld_ug, void* out, long long ldo, int L, int F, void* stream);

#ifdef __cplusplus
}
#endif

#endif  // YUME_B200_T5_H_
