/* yume_b200_fp8_attn.h — C ABI of the FP8 (e4m3) self-attention of precision="fp8_attn" in libyume_b200.so (conventions as
 * include/yume_b200.h: device pointers, `stream` a cudaStream_t as void*, no allocation, no synchronisation, capture-safe
 * launches, 0 or a negative YB_ERR_* code).
 *
 * Numerics (every entry point below and the torch twins in the test-suite implement exactly this):
 *   Q, K     after RMSNorm + RoPE, one yb_quant_rows_fp8 launch (include/yume_b200_fp8.h) over the [L, 2C] view qkv[:, :2C] of the
 *            fused q|k|v rows: a 1x128 group is one head of one token, so the scale table f32 [2 heads, lds] holds the q scale
 *            of head h at row h and the k scale of head h at row heads + h.
 *   V        per (head, 128-key tile): amax over the 128 x 128 block (NaN ignored), inv = 448 / amax (IEEE fp32 division),
 *            s_v = amax / 448, q = cvt.rn.satfinite.e4m3(v * inv); when 448 / amax is not finite the block is zeros with
 *            s_v = 0 (the 1x128 rules of include/yume_b200_fp8.h, applied to a 128 x 128 block). Stored transposed,
 *            vt8 e4m3 [heads, 128, Lkp] with Lkp = ceil(Lk / 128) * 128, keys >= Lk as zeros, and within every 32-key block
 *            in the order pi(f) = 16 floor(f / 16) + 2 floor((f mod 16) / 4) + 8 floor((f mod 4) / 2) + (f mod 2):
 *            vt8[h, d, 32 b + f] = q(V[32 b + pi(f), h 128 + d]).  s_v f32 [heads, Lkp / 128].
 *            pi makes the fp32 accumulator fragment of S hold, in every thread, exactly the keys its 8-bit A fragment of
 *            m64nNk32 needs (rows r and r + 8, k = 4 (lane % 4) + {0..3} and + 16), so P packs to e4m3 inside the thread.
 *   Attention  non-causal, softmax scale `scale` (1 / sqrt(128) in the engine), keys >= Lk masked. Per 128-key tile j:
 *            S = Q8 K8_j^T as four wgmma m64n128k32 e4m3 into a fresh accumulator, x = S s_k[key] s_q[row] scale log2(e)
 *            (the row factor folded into the exp2 FFMA), online softmax in fp32 (running max m, l summing the unrounded p),
 *            P8 = e4m3(256 p) computed as 2^(x - m + 8), O_tile = P8 Vt8_j as four wgmma into a fresh accumulator, then
 *            O = O alpha + O_tile s_v[j] / 256 in fp32 (promotion: the e4m3 tensor-core accumulator keeps 13 mantissa bits).
 *            out = O / l as bf16.
 */
#ifndef YUME_B200_FP8_ATTN_H_
#define YUME_B200_FP8_ATTN_H_

#include "yume_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------------
 * v bf16 [Lk, heads * 128] (row stride ldv elements, % 8; 16-byte aligned) -> vt8 e4m3 [heads, 128, Lkp] (dense, 16-byte
 * aligned) + v_scale f32 [heads, Lkp / 128] (dense). One CTA per (head, 128-key tile).
 * ------------------------------------------------------------------------------------------- */
int yb_quant_vt_fp8(const void* v, long long ldv, void* vt8, void* v_scale, int Lk, int heads, void* stream);

/* ---------------------------------------------------------------------------------------------
 * out bf16 [Lq, heads * 128] (row stride ldo, % 8) = softmax(Q K^T scale) V of the quantised operands above.
 *   q8         e4m3 [Lq, heads * 128], row stride ldq bytes (% 16)
 *   k8         e4m3 [Lk, heads * 128], row stride ldk bytes (% 16)
 *   qk_scale   f32 [2 heads, lds] (q scales, then k scales), lds % 4 == 0, lds >= Lq and >= Lk
 *   vt8, v_scale   as yb_quant_vt_fp8 writes them for the same Lk and heads
 *   flags      only the KV split policy bits (YB_ATT_SPLIT_SHIFT, as yb_attention); anything else is YB_ERR_ARG
 *   ws         the tail split's workspace: yb_attention_workspace_bytes(Lq, Lk, heads, sms, flags) bytes, as for yb_attention
 *              (NULL or too small: the launch is not split)
 * Same work decomposition (yb_attention_plan), workspace and combine as yb_attention: 256-row units run as two 128-row query
 * tiles by one TMA producer and two consumer warpgroups.
 * ------------------------------------------------------------------------------------------- */
int yb_attention_fp8(const void* q8, long long ldq, const void* k8, long long ldk, const void* qk_scale, long long lds,
                     const void* vt8, const void* v_scale, void* out, long long ldo, int Lq, int Lk, int heads, float scale,
                     int flags, void* ws, long long ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif

#endif  // YUME_B200_FP8_ATTN_H_
