/* yume_b200_fp8_sp.h — C ABI of the pieces that run precision="fp8" and "fp8_attn" under Ulysses sequence parallelism in
 * libyume_b200.so (conventions as include/yume_b200.h: device pointers, `stream` a cudaStream_t as void*, no allocation, no
 * synchronisation, capture-safe launches, 0 or a negative YB_ERR_* code).
 *
 * A 1x128 activation scale group is one head of one token (head_dim 128), so quantising q, k or the attention output gives the same
 * values and scales on whichever rank holds that head. The entry points below are the one-GPU fp8 kernels with the layouts of the
 * Ulysses exchange; their numerics are those of include/yume_b200_fp8.h and include/yume_b200_fp8_attn.h, bit for bit:
 *   yb_quant_rows_fp8_split   == yb_quant_rows_fp8 of the gathered [M, K] matrix
 *   yb_attention_fp8_sp       == yb_attention_fp8 for the same operands and flags; only the address of each stored row differs
 *   yb_sp_pack_qkv            == the NCCL send buffer that the bf16 engine builds with the n_split q|k|v GEMM and
 *                                yb_qk_norm_rope (pieces), for the same bf16 q|k|v rows
 */
#ifndef YUME_B200_FP8_SP_H_
#define YUME_B200_FP8_SP_H_

#include "yume_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------------
 * yb_quant_rows_fp8 with a K-split source: logical column k of row m is x[(k / split) * split_stride + m * ldx + k % split]
 * (the [P, Lp, heads/P * 128] attention output the Ulysses exchange delivers, read as [Lp, C]; the layout yb_gemm_bf16 reads
 * through a_split). -> e4m3 [M, K] (row stride ldo bytes, % 16) + f32 scales [K / 128, lds].
 * Constraints: K % 128 == 0 and split % 128 == 0 and K % split == 0 (YB_ERR_SHAPE); ldx, split_stride % 8; 16-byte aligned x
 * and out; lds % 4 and >= M.
 * ------------------------------------------------------------------------------------------- */
int yb_quant_rows_fp8_split(const void* x, long long ldx, int split, long long split_stride, void* out, long long ldo,
                            void* out_scale, long long lds, int M, int K, void* stream);

/* ---------------------------------------------------------------------------------------------
 * yb_attention_fp8 (include/yume_b200_fp8_attn.h) whose epilogue stores output row g (of Lq = world * Lp gathered query rows)
 * into row rank * Lp + g % Lp of out_peers[g / Lp] (a [world(src), Lp, heads * 128] receive buffer on each rank, row stride
 * ldo elements), as yb_attention_sp does. The tail split's combine scatters the same way. Same plan, workspace and flags as
 * yb_attention_fp8. Constraints: 2 <= world <= 8, 0 <= rank < world, Lq == world * Lp, Lk <= Lq.
 * ------------------------------------------------------------------------------------------- */
int yb_attention_fp8_sp(const void* q8, long long ldq, const void* k8, long long ldk, const void* qk_scale, long long lds,
                        const void* vt8, const void* v_scale, void* const* out_peers, long long ldo, int Lq, int Lk, int heads,
                        float scale, int world, int rank, int Lp, int flags, void* ws, long long ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * The NCCL send side of the Ulysses q|k|v exchange: yb_sp_scatter_qkv's arithmetic (RMSNorm over all C columns of q and of k,
 * times the norm weight, RoPE on rows < rope_len; v copied) with this rank's own send buffer as destination. qkv bf16 [L, 3C]
 * (row stride ld) -> send bf16 [world(owner), Lp, 3 Wh] (dense, Wh = C / world): the q | k | v columns of the heads of rank p go
 * to send[p, row, 0:Wh | Wh:2Wh | 2Wh:3Wh]. L <= Lp. Constraints as yb_sp_scatter_qkv.
 * ------------------------------------------------------------------------------------------- */
int yb_sp_pack_qkv(const void* qkv, long long ld, const void* wq, const void* wk, const void* rope, int rope_len, int L, int C,
                   int D, float eps, void* send, int world, int Lp, void* stream);

#ifdef __cplusplus
}
#endif

#endif  // YUME_B200_FP8_SP_H_
