/* yume_b200.h — C ABI of libyume_b200.so: the H100 (sm_90a) kernels behind YUME's denoise hot path.
 *
 * The reference (stdstu12/YUME) has no FFI: its extension seam is Python method re-binding on the
 * WanModel instance (wan23/textimage2video.py:190-194) plus the module-level function
 * `flash_attention` (wan23/modules/attention.py:24-38). This C ABI sits *under* those seams: the Python
 * host side (yume_b200/*.py) keeps the reference's call signatures and hands raw device pointers to the
 * entry points below. Each entry point names the reference code it replaces.
 *
 * Conventions: every pointer is a CUDA device pointer unless stated; `stream` is a cudaStream_t passed as
 * void*; functions never allocate device memory, never synchronise, never throw (workspaces are caller-owned); they return 0 on
 * success or a negative YB_ERR_* code. Row-major everywhere, strides in elements.
 */
#ifndef YUME_B200_H_
#define YUME_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define YB_OK 0
#define YB_ERR_ARG (-1)        /* null pointer / out-of-range enum / non-positive size */
#define YB_ERR_SHAPE (-2)      /* shape not supported by the kernel (see each function) */
#define YB_ERR_ALIGNMENT (-3)  /* pointer or stride not 16-byte aligned */
#define YB_ERR_NO_DRIVER (-4)  /* cuTensorMapEncodeTiled not available (no CUDA driver) */
#define YB_ERR_TENSORMAP (-5)  /* driver rejected a TMA descriptor */
#define YB_ERR_LAUNCH (-6)     /* kernel launch failed (message on stderr) */

/* ABI version: bump on any signature change. */
int yb_abi_version(void);

/* ---------------------------------------------------------------------------------------------
 * GEMM with fused epilogue: out = epi(A[M,K] * B[N,K]^T + bias[N]); A, B bf16; fp32 accumulate (wgmma).
 * Replaces nn.Linear q/k/v/o (wan23/modules/model.py:171-174,190-192,206), ffn (:265-267,309-312),
 * text_embedding (:455-457), cross-attn projections (:222-224,231) and the patch-embedding Conv3d
 * (kernel==stride, :453-454) after yb_patchify has gathered the patches.
 * Constraints: N % 32 == 0, K % 8 == 0, lda/ldb % 8 == 0, ldo % 8 == 0; A, B, out 16-byte aligned.
 * ------------------------------------------------------------------------------------------- */
#define YB_EPI_BF16 0      /* out bf16 = acc + bias */
#define YB_EPI_GELU_BF16 1 /* out bf16 = gelu_tanh(acc + bias)            (nn.GELU(approximate='tanh')) */
#define YB_EPI_F32 2       /* out f32  = acc + bias */
#define YB_EPI_GATE_RES 3  /* out f32 += (acc + bias) * gate[tok_idx[m]][n]   (model.py:304,308,312) */
#define YB_EPI_RES_BF16 5  /* out bf16 = acc + bias + res[m][n]  (ResnetBlockCausal3D skip add, unet_causal_3d_blocks.py:413;
                              diffusers Attention residual_connection) */
#define YB_EPI_GELU_ERF_BF16 4 /* out bf16 = gelu_erf(acc + bias)         (nn.GELU() in MLPProj, wan/modules/model.py:536) */

typedef struct yb_gemm_args {
  unsigned int struct_bytes; /* = sizeof(yb_gemm_args): the library rejects a caller built against another layout */
  int cta_pair;    /* kernel choice: 0 = automatic (the 1-CTA kernel: the faster form on the H100, see yb_gemm_plan), 1 = the 1-CTA
                      kernel, 2 = the SM-pair kernel (a 2-CTA cluster per 256-row tile, B operand multicast) */
  const void* A;   /* bf16 [M, K], row stride lda */
  const void* B;   /* bf16 [N, K], row stride ldb  (nn.Linear.weight layout) */
  const void* bias;/* f32 [N] or NULL */
  void* out;       /* bf16/f32 [M, N] row stride ldo; for YB_EPI_GATE_RES the fp32 residual stream, updated in place */
  const void* gate;    /* YB_EPI_GATE_RES: f32 [U, gate_ld] gate table or NULL (gate == 1, cross-attention) */
  const void* tok_idx; /* YB_EPI_GATE_RES: int32 [M] row of `gate` per token, or NULL (all tokens use row 0) */
  long long lda, ldb, ldo, gate_ld;
  int M, N, K;
  int epilogue;    /* YB_EPI_* */
  int block_n;     /* N tile: 0 = auto; 1-CTA kernel 128 / 256; SM-pair kernel any multiple of 32 up to 256 (auto: 256, or N rounded
                      up to 32 when N < 256) */
  int n_split;     /* YB_EPI_BF16 only: > 0 => output column block j (width n_split, % 32 == 0) is written at
                      out + j*split_stride + m*ldo + (n % n_split): the peer-major layout the Ulysses all-to-all sends */
  long long split_stride;
  int a_split;     /* > 0 => A is K-split: logical column k is element (k % a_split) of chunk k / a_split, chunks
                      a_split_stride elements apart (the [P, L/P, heads/P*128] buffer an Ulysses all-to-all delivers);
                      a_split % 64 == 0, K % a_split == 0. 0 => ordinary [M, K] matrix. */
  long long a_split_stride;
  const void* res;  /* YB_EPI_RES_BF16: bf16 [M, N] residual, row stride res_ld */
  long long res_ld;
  /* Tail split-K (SM-pair kernel, YB_EPI_GATE_RES): when the last wave of output tiles fills at most part of the SM pairs (the
   * per-rank shapes of multi-GPU Ulysses), its tiles are cut into K segments that run as separate work
   * items and leave fp32 partials in `ws`; a second kernel adds them and applies the epilogue. split_k: 0 = automatic,
   * 1 = never, 2..12 = force that many segments on the last wave (tests). ws / ws_bytes: CALLER-owned workspace of at least
   * yb_gemm_workspace_bytes(...) bytes, 16-byte aligned; NULL or too small = the launch is simply not split (same result up to
   * fp32 summation order). The library never allocates. */
  int split_k;
  void* ws;
  long long ws_bytes;
} yb_gemm_args;
int yb_gemm_bf16(const yb_gemm_args* args, void* stream);
long long yb_gemm_workspace_bytes(int M, int N, int K, int epilogue, int cta_pair, int split_k);
/* Host-only: out3 = {whole tiles, K segments per tail tile (1 = no split), 64-column K blocks per segment}. */
int yb_gemm_splitk_plan(int tiles, int num_kb, int clusters, int split_k, int* out3);
/* Host-only: the kernel / tiling yb_gemm_bf16 picks for an [M, N] output on a GPU with `sms` SMs (no device access).
 * out4 = {1 if the SM-pair kernel, N tile, M tiles (of 256 rows for the pair kernel, 128 otherwise), N tiles}. */
int yb_gemm_plan(int M, int N, int sms, int* out4);

/* ---------------------------------------------------------------------------------------------
 * CausalConv3d k=3 (replicate pad W 1,1 / H 1,1 / T 2,0 then Conv3d: hyvideo/vae/unet_causal_3d_blocks.py:48-74) as an
 * implicit GEMM on wgmma: out[voxel, co] = bias[co] + sum_{tap,ci} xpad[t+dt, h+dh, w+dw, ci] * w[co, tap*Cp + ci].
 *   xpad  bf16 [T+2, H+2, W+2, Cp] channels-last, already replicate-padded (yb_vae_pad_act writes it), Cp % 64 == 0
 *   w     bf16 [Cout, 27*Cp], tap = (dt*3 + dh)*3 + dw (Conv3d weight permuted to [co, kt, kh, kw, ci]); Cout % 32 == 0
 *   out   [T*H*W, ldo] channels-last; epilogue YB_EPI_BF16, YB_EPI_F32 or YB_EPI_RES_BF16 (+ res bf16 [T*H*W, res_ld])
 * ------------------------------------------------------------------------------------------- */
typedef struct yb_conv3d_args {
  unsigned int struct_bytes; /* = sizeof(yb_conv3d_args) */
  int cta_pair;              /* SM-pair kernel (each CTA of a cluster owns one 128-voxel box, the weight tile is split between the two,
                                un-fused taps): 1 = always; 0 (automatic) and 2 = the 1-CTA kernel */
  const void* xpad;
  const void* w;
  const void* bias; /* f32 [Cout] or NULL */
  void* out;
  const void* res;
  long long ldo, res_ld;
  int T, H, W, Cp, Cout;
  int epilogue;
  /* Generalisations used by the Wan2.2 VAE (wan23/modules/vae2_2.py); all-zero = the 3x3x3 replicate-padded form above.
   *   kt, kh, kw     taps per axis, each 1 or 3 (0 = 3): Conv2d 3x3 is (1,3,3), Resample.time_conv is (3,1,1)
   *   oob_zero_pad   1: `xpad` is the UNPADDED [T, H, W, Cp] activation and the causal zero padding (kt-1 in front,
   *                  kh/2, kw/2 around; vae2_2.py:22-44) is TMA out-of-bounds zero fill — no padded buffer exists
   *   out_t_mul/add  output frame of input frame t is t*out_t_mul + out_t_add (0 = identity): interleaves the two
   *                  channel groups of time_conv into consecutive frames (vae2_2.py:151-154)
   *   fuse_w         tile-shape policy for kw == 3: 0 = automatic, 1 = never, 2 = always use the kw-fused kernel (one
   *                  130-voxel TMA halo row feeds all three kw taps through row-shifted UMMA descriptors); results are
   *                  identical either way — the knob exists for tests and profiling */
  int kt, kh, kw;
  int oob_zero_pad;
  int out_t_mul, out_t_add;
  int fuse_w;
  /* Strided form, the `Resample` convs of Encoder3d (wan23/modules/vae2_2.py:101-110, 158-170; wan/modules/vae.py:84-90, 125-139);
   * needs oob_zero_pad. T, H, W stay the INPUT extents; out has To*Ho*Wo rows.
   *   stride_hw  2: Conv2d(3x3, stride 2) behind ZeroPad2d((0,1,0,1)) — no padding in front, one zero row/column behind:
   *              Ho = (H + 1 - kh) / 2 + 1, Wo likewise; output (ho, wo) reads input rows 2ho .. 2ho+2
   *   stride_t   2: time_conv CausalConv3d((3,1,1), stride (2,1,1), padding 0) over the frames it is given:
   *              To = (T - kt) / 2 + 1; output t reads input frames 2t .. 2t+2
   * 0 or 1 = unit stride. The tensor map samples every second voxel, so no padded or gathered copy of the input exists. */
  int stride_t, stride_hw;
} yb_conv3d_args;
int yb_conv3d_causal(const yb_conv3d_args* args, void* stream);
/* Host-only: the tile plan yb_conv3d_causal would use (no device access; pins the chooser in the CPU test-suite).
 * out4 = {TW, TH, TT, kw-fused?}: the 128-voxel output tile is a TT x TH x TW box; fused = one-row tile + 130-voxel halo. */
int yb_conv3d_plan(int T, int H, int W, int Cout, int kw, int fuse_w, int* out4);

/* ---------------------------------------------------------------------------------------------
 * Fused LayerNorm (no affine, eps) + adaLN modulate -> bf16:  h = LN(x) * (1 + scale) + shift
 * Replaces WanLayerNorm.forward + `norm1(x).float() * (1 + e[1]) + e[0]` (wan23/modules/model.py:140-150,
 * 301,310; 14B: wan/modules/model.py:470-476). With `weight`/`lnbias` non-NULL and scale/shift NULL it is
 * the affine norm3 in front of cross-attention (:259-261,308).
 *   x      f32 [L, C]            scale/shift: f32 rows of a [U, mod_ld] table, selected per token by tok_idx
 *   out    bf16 [L, ldo] (out_f32 == 0) or f32 [L, ldo] (out_f32 == 1, used by Head: model.py:343-347)
 * Constraints: C % 8 == 0, C <= 8192.
 * ------------------------------------------------------------------------------------------- */
int yb_ln_modulate(const void* x, long long ldx, void* out, long long ldo, int out_f32, const void* scale,
                   const void* shift, long long mod_ld, const void* tok_idx, const void* weight, const void* lnbias,
                   int L, int C, float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fused WanRMSNorm (over the full C row, fp32 math) + weight + 3-axis RoPE, in place on bf16 rows.
 * Replaces WanRMSNorm.forward (wan23/modules/model.py:121-137) and rope_apply (:38-118) for q and k.
 *   qk     bf16, rows of C elements at qk + t*ld (t < L); normalised, scaled by weight[C] (f32) and,
 *          when `rope` != NULL, rotated: pair j of every head uses (cos,sin) = rope[t][j] (f32 [L, D/2, 2]);
 *          tokens t >= rope_len are left un-rotated (model.py:73).
 * Constraints: C % 8 == 0, head_dim D even, C % D == 0.
 * ------------------------------------------------------------------------------------------- */
int yb_rmsnorm_rope(void* qk, long long ld, const void* weight, const void* rope, int rope_len, int L, int C, int D,
                    float eps, void* stream);
/* Same with the C columns of a row stored in pieces: column c is element (c % piece_cols) of piece c / piece_cols,
 * pieces piece_stride elements apart (peer-major Ulysses send buffer). piece_cols % 8 == 0, C % piece_cols == 0. */
int yb_rmsnorm_rope_pieces(void* qk, long long ld, int piece_cols, long long piece_stride, const void* weight,
                           const void* rope, int rope_len, int L, int C, int D, float eps, void* stream);

/* q AND k of the same token rows in ONE launch (WanSelfAttention runs norm_q(q), norm_k(k) and rope_apply on both with the
 * same per-token angles, wan23/modules/model.py:190-200): q, k point at the first element of the two [L, C] row sets (same
 * row stride ld, same piece layout as yb_rmsnorm_rope_pieces; piece_cols = C, piece_stride = 0 for plain rows). */
int yb_qk_norm_rope(void* q, void* k, long long ld, int piece_cols, long long piece_stride, const void* wq, const void* wk,
                    const void* rope, int rope_len, int L, int C, int D, float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Non-causal softmax(Q K^T * scale) V, head_dim 128, bf16 in / bf16 out, fp32 softmax + accumulate.
 * Replaces flash_attention(q, k, v, k_lens=...) (wan23/modules/attention.py:24-130) for B == 1.
 *   q: bf16 [Lq, heads*128] at row stride ldq (head h = columns [h*128, h*128+128)); k, v likewise with Lk rows.
 *   Keys >= Lk are masked (the k_lens contract, attention.py:74-81). out: bf16 [Lq, heads*128] stride ldo.
 * Constraints: head_dim == 128; strides % 8 == 0; pointers 16-byte aligned.
 * ------------------------------------------------------------------------------------------- */
int yb_attention(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* out,
                 long long ldo, int Lq, int Lk, int heads, float scale, int flags, void* stream);
/* Full form. `ws` / `ws_bytes`: caller-owned device workspace for the automatic KV tail split (size it with
 * yb_attention_workspace_bytes; NULL or too small = the launch is not split — same result, a partly idle last wave; the
 * library itself never allocates and never synchronises, so the call is CUDA-graph-capture safe). `trace`: ignored (kept so that
 * callers built against earlier versions of this header still link); pass NULL. */
int yb_attention_ex(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* out,
                    long long ldo, int Lq, int Lk, int heads, float scale, int flags, void* ws, long long ws_bytes,
                    void* trace, void* stream);
#define YB_ATT_P_SMEM 1     /* flags bit 0: stage P through shared memory instead of registers (debug variant) */
#define YB_ATT_EMU_SHIFT 2  /* flags bits 2-3: retired (FMA-pipe exponentials: measured slower in rounds 1 and 2, removed); must be 0 */
#define YB_ATT_ACCUMULATE 2 /* flags bit 1: out += result (WanI2VCrossAttention sums the text and image branches,
                               wan/modules/model.py:380-387) */
#define YB_ATT_SPLIT_SHIFT 4 /* flags bits 4-6: KV split policy. 0 = automatic (the units of a last wave that is at most
                               half full are cut into KV segments and merged by a combine kernel), 1 = never, 2..4 = cut
                               EVERY unit into that many segments (tests). Results are identical up to fp32 rounding. */
/* Host-only: the work decomposition yb_attention would use on a GPU with `sms` SMs (no device access; the CPU test-suite
 * pins the scheduler with it). out4 = {CTAs running whole units, tail units that are split, KV segments per tail unit,
 * 128-key tiles per segment}. flags as for yb_attention (ACCUMULATE disables the split; bits 4-6 force it). */
int yb_attention_plan(int Lq, int Lk, int heads, int sms, int flags, int* out4);
/* Host-only: bytes of workspace yb_attention_ex / yb_attention_sp need for that decomposition (0 when nothing is split). */
long long yb_attention_workspace_bytes(int Lq, int Lk, int heads, int sms, int flags);
/* Test hook: force the KV split policy (0 = off, 1..4 as YB_ATT_SPLIT_SHIFT) for every later launch whose flags leave it
 * automatic — lets the multi-GPU parity tool drive the split + peer-scatter combine path. Process-global, not thread-safe. */
int yb_debug_force_split(int ns);
/* ---------------------------------------------------------------------------------------------
 * Ulysses sequence parallelism fused with the NVLink exchange (SURVEY.md §8e; design reference
 * wan23/distributed/ulysses.py:9-47, sequence_parallel.py:147-176 — three NCCL all_to_alls in, one out).
 * `peers[r]` are device pointers valid on THIS GPU to rank r's receive buffer (CUDA peer / symmetric memory).
 *   yb_sp_scatter_qkv: per local token, RMSNorm+weight+RoPE on q and k (WanRMSNorm over all heads, model.py:121-137;
 *     rope_apply :38-118), then every 16-byte chunk of q|k|v is stored into the receive buffer of the rank owning
 *     that head: peers[h / (heads/P)][rank][t][part*Wh + ...], buffer layout [P(src), Lp, 3*Wh], Wh = C/P.
 *   yb_attention_sp: attention over the gathered tokens for this rank's heads; output row g is stored into
 *     out_peers[g / Lp][rank][g % Lp][:], buffer layout [P(src), Lp, heads_local*128] (row stride ldo).
 * A cross-rank barrier (symmetric-memory signal) must separate each call from the consumer of the buffers.
 * ------------------------------------------------------------------------------------------- */
int yb_sp_scatter_qkv(const void* qkv, long long ld, const void* wq, const void* wk, const void* rope, int rope_len,
                      int L, int C, int D, float eps, void* const* peers, int world, int rank, int Lp, void* stream);
/* GEMM + collective in ONE kernel (the second Ulysses transport, "p2p_gemm"): the fused q|k|v projection of this rank's Lp_rows
 * local tokens (A bf16 [Lp_rows, K], W bf16 [3C, K] = q|k|v weights stacked, bias f32 [3C]) on the SM-pair wgmma kernel whose
 * EPILOGUE is the all-to-all: the columns of head h are stored straight into the receive buffer of the rank that owns h
 * (`peers[r]`, layout [P(src), Lp, q|k|v of heads/P] as for yb_sp_scatter_qkv), so the NVLink transfer rides under the GEMM's
 * main loop instead of a separate pass. WanRMSNorm spans all heads of a token, which no single receiver holds: the epilogue
 * also accumulates the per-token sums of squares of the (bf16-rounded) q and k columns into `sums` f32 [Lp][2] (atomics; the
 * caller zeroes it once, yb_sp_bcast_sums re-zeroes it), yb_sp_bcast_sums copies them into slot `rank` of every peer's
 * [P, Lp, 2] table, and — after the cross-rank barrier — yb_sp_post_norm_rope finishes q, k in place on the RECEIVED rows:
 * bf16(rope(x * rstd(token) * weight[my heads])), the arithmetic of yb_rmsnorm_rope moved behind the exchange. */
int yb_gemm_sp_qkv(const void* A, long long lda, const void* W, const void* bias, int Lp_rows, int C, int K, void* const* peers,
                   int world, int rank, int Lp, void* sums, void* stream);
int yb_sp_bcast_sums(void* local_sums, void* const* peer_tables, int world, int rank, int Lp, void* stream);
int yb_sp_post_norm_rope(void* buf, const void* sums, const void* wq, const void* wk, const void* rope, int rope_len, int L,
                         int Wh, int C, int D, float eps, void* stream);
int yb_attention_sp(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                    void* const* out_peers, long long ldo, int Lq, int Lk, int heads, float scale, int world, int rank,
                    int Lp, int flags, void* ws, long long ws_bytes, void* stream);   /* flags / ws as yb_attention_ex */

/* ---------------------------------------------------------------------------------------------
 * patchify gather (bit-exact index op): x f32 [Cin, F, H, W] (element strides sc, sf, sh, sw) -> bf16 [F*(Hp)*(Wp), Cin*ph*pw] rows in
 * (f, h, w) token order, columns in Conv3d weight order (cin, ph, pw); H, W zero-padded up to a multiple
 * of the patch (convpadd, wan23/modules/model.py:918-931). Replaces the data movement of
 * `patch_embedding(u).flatten(2).transpose(1, 2)` (:750-753); the contraction itself is yb_gemm_bf16.
 * ------------------------------------------------------------------------------------------- */
int yb_patchify(const void* x, long long sc, long long sf, long long sh, long long sw, void* out, long long ldo,
                int Cin, int F, int H, int W, int ph, int pw, void* stream);

/* unpatchify (bit-exact): y f32 [L, ph*pw*Cout] (row stride ldy) -> out f32 [Cout, F, Hp*ph, Wp*pw]
 * (einsum 'fhwpqrc->cfphqwr', wan23/modules/model.py:867-890; patch_t == 1). */
int yb_unpatchify(const void* y, long long ldy, void* out, int Cout, int F, int Hp, int Wp, int ph, int pw,
                  void* stream);

/* out[r1][r2][:] = a[r1][:] + b[r2][:] (f32): per-block adaLN tables `modulation + e0` (wan23/modules/model.py:296,344). */
int yb_bcast_add(const void* a, const void* b, void* out, int R1, int R2, int n, void* stream);

/* Sinusoidal timestep embedding in fp64 -> f32 [n, dim] = [cos | sin] (wan23/modules/model.py:14-24). t: f32 [n]. */
int yb_sinusoidal(const void* t, void* out, int n, int dim, void* stream);

/* Small-M fp32 linear: out[M,N] = act(in[M,K]) * W[N,K]^T + bias, act = SiLU if silu_in (M <= 16).
 * Replaces time_embedding / time_projection under autocast(fp32) (wan23/modules/model.py:459-461,805-812). */
int yb_linear_f32_small(const void* in, const void* W, const void* bias, void* out, int M, int N, int K, int silu_in,
                        void* stream);

/* General fp32 linear (SIMT, exact fp32): out[M,N] = in[M,K] * W[N,K]^T + bias. Replaces Head.head
 * (wan23/modules/model.py:331,346) which the reference runs under autocast(fp32). N % 4 == 0, K % 4 == 0, ldi % 4 == 0
 * (YB_ERR_SHAPE otherwise); in and W 16-byte aligned (YB_ERR_ALIGNMENT otherwise). */
int yb_linear_f32(const void* in, long long ldi, const void* W, const void* bias, void* out, long long ldo, int M,
                  int N, int K, void* stream);

/* ---------------------------------------------------------------------------------------------
 * VAE decoder glue (hyvideo/vae; channels-last bf16 activations [T*H*W, C]).
 * ------------------------------------------------------------------------------------------- */
/* GroupNorm statistics: stats f64 [G][2] += (sum, sum of squares) per group over x bf16 [N, C] (row stride ld).
 * Caller zeroes `stats`. (nn.GroupNorm(32, C, eps=1e-6): unet_causal_3d_blocks.py:299,323; vae.py:204) */
int yb_gn_stats(const void* x, long long ld, void* stats, long long N, int C, int G, void* stream);
/* One gather pass: [GroupNorm apply (stats, gamma, beta) ->] [SiLU ->] nearest upsample (ft in {1,2}; fh, fw) ->
 * replicate padding (pad=1: out bf16 [T+2, H+2, W+2, Cp], temporal pad 2 in front; pad=0: out [T, H, W, Cp]) where
 * (T, H, W) = (ft==2 ? 1+2(Ts-1) : Ts, Hs*fh, Ws*fw) and the first frame is only upsampled spatially
 * (UpsampleCausal3D :156-163; CausalConv3d padding :61-62,73; ResnetBlockCausal3D norm+act :375-379,401-409). */
int yb_vae_pad_act(const void* x, long long ldx, int Ts, int Hs, int Ws, int C, void* out, int Cp, int pad, int ft, int fh,
                   int fw, const void* stats, const void* gamma, const void* beta, int G, float eps, int silu,
                   void* stream);
/* Frame-causal softmax of attention scores S f32 [L, ldS] -> P bf16 [L, ldP]: row i keeps keys j < (i/hw + 1)*hw
 * (prepare_causal_attention_mask :37-45; upcast softmax of the diffusers Attention). */
int yb_masked_softmax(const void* S, long long ldS, void* P, long long ldP, int L, int hw, void* stream);
/* z f32 [Cn, N] (NCDHW, N = T*H*W) -> bf16 [N, ldo] channels-last (columns >= Cn zero), and back for f32. */
int yb_nchw_to_nhwc_bf16(const void* x, void* out, long long N, int Cn, int ldo, void* stream);
int yb_nhwc_to_nchw_f32(const void* x, long long ldx, void* out, long long N, int Cn, void* stream);
/* Same with clamp to [lo, hi] fused: the tail of `WanVAE.decode` (wan/modules/vae.py:655-663: head conv output ->
 * `.float().clamp_(-1, 1)`) on the channels-last f32 head output. */
int yb_nhwc_to_nchw_f32_clamp(const void* x, long long ldx, void* out, long long N, int Cn, float lo, float hi, void* stream);
/* Tile cross-fade (blend_v / blend_h / blend_t, autoencoder_kl_causal_3d.py:343-359) on contiguous f32 tiles:
 * b[o, y, i] = a[o, ea-ext+y, i] * (1 - y/ext) + b[o, y, i] * (y/ext) for y < ext; a is [outer, ea, inner], b [outer, eb, inner].
 * Bit-exact with the reference's expression on f32 tensors: the weights are computed in double and rounded to f32, and each
 * product and the sum is rounded on its own (no fused multiply-add), as in yb_vae_assemble_tiles. */
int yb_blend(const void* a, void* b, long long outer, int ea, int eb, int ext, long long inner, void* stream);

/* One-pass assembly of a tiled decode (temporal_tiled_decode / spatial_tiled_decode + blend_v / blend_h / blend_t,
 * autoencoder_kl_causal_3d.py:343-359, 417-463, 500-531): the final f32 [C, F, H, W] video straight from the RAW decoded tiles — each
 * output voxel is the reference's in-place cross-fade sequence written out as one expression of <= 2 x 4 raw tile values (same
 * operations, same order, bit for bit: weights rounded from double, products and sums rounded separately as torch does), so tiles
 * may be decoded in any order / on any GPU and no torch.cat or per-row blend launch remains. Exact when no tile is read back inside
 * its own blended region: every interior tile k of a row / column / window sequence has size >= ext(k) + ext(k+1), ext(k) = the
 * clamped blend extent with its predecessor (tile overlap factors <= 0.5 always satisfy this).
 *   tile_ptrs  DEVICE array [nt*ni*nj] of device pointers: tile (ti, i, j) = f32 [C, tlen[ti] + tskip(ti), th[i], tw[j]] contiguous,
 *              tskip(ti) = 1 for ti > 0 (the first decoded frame of later temporal tiles is dropped, :519-520), else 0
 *   th, tw, tlen, tf0   DEVICE int arrays: tile heights [ni] / widths [nj] in pixels, kept-length source frames [nt] (after the
 *              drop), first output frame [nt]
 *   row_limit / blend_extent (space), t_limit / t_blend_extent (time): the reference's crop and cross-fade lengths */
int yb_vae_assemble_tiles(const void* const* tile_ptrs, const int* th, const int* tw, const int* tlen, const int* tf0, int nt,
                          int ni, int nj, int C, int F, int H, int W, int row_limit, int blend_extent, int t_limit,
                          int t_blend_extent, void* out, void* stream);

/* Wan2.2 VAE decoder glue (wan23/modules/vae2_2.py), channels-last bf16:
 *   yb_vae_rms_act: out[T, Hs*up, Ws*up, Cp] = [SiLU]([RMS_norm over channels * gamma](x)) nearest-exact upsampled by
 *     `up` in {1,2} (RMS_norm :47-61 = F.normalize * sqrt(C) * gamma; Upsample :64-70). gamma NULL = no norm.
 *   yb_vae_dupup_add: main += DupUp3D(x) over the whole frame sequence, first ft-1 duplicated frames dropped
 *     (:376-418, :499-503). main bf16 [ft*Ts-(ft-1), Hs*fs, Ws*fs, out_c], x bf16 [Ts, Hs, Ws, in_c], both dense.
 *   yb_vae_unpatchify2_clamp: y f32 [T*H*W, ldy] (12 channels) -> out f32 [3, T, 2H, 2W] clamped to [-1,1]
 *     (unpatchify :305-319; Wan2_2_VAE.decode :1066-1067). */
int yb_vae_rms_act(const void* x, long long ldx, void* out, const void* gamma, int T, int Hs, int Ws, int C, int Cp, int up,
                   int silu, void* stream);
int yb_vae_dupup_add(void* main_, const void* x, int Ts, int Hs, int Ws, int in_c, int out_c, int ft, int fs, void* stream);
int yb_vae_unpatchify2_clamp(const void* y, long long ldy, void* out, int T, int H, int W, void* stream);
/* Wan2.2 VAE ENCODER glue (SURVEY.md §8(f) rank 3; `Wan2_2_VAE.encode`, vae2_2.py:796-829):
 *   yb_vae_avgdown_add: main += AvgDown3D(x) over the whole frame sequence (:320-373, :449-459): (ft - T % ft) % ft zero frames
 *     in front, (c, a, q, r) flattened and averaged in groups of in_c*ft*fs*fs / out_c. x bf16 [T, H, W, in_c],
 *     main bf16 [ceil(T/ft), H/fs, W/fs, out_c], both dense; H, W divisible by fs.
 *   yb_vae_patchify2_bf16: video f32 [3, T, H, W] -> out bf16 [T*(H/2)*(W/2), ldo], 12 channels (c r q) (:284-300), the other
 *     ldo - 12 columns zeroed. */
int yb_vae_avgdown_add(void* main_, const void* x, int T, int H, int W, int in_c, int out_c, int ft, int fs, void* stream);
int yb_vae_patchify2_bf16(const void* video, void* out, long long ldo, int T, int H, int W, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Self-test of the wgmma / TMA building blocks on one 128x128x128 tile (used by tests/, not by the product path).
 *   mode 0: A smem K-major, B smem K-major        D = A[128,128] * Bk[128(n),128(k)]^T
 *   mode 1: A smem K-major, B smem MN-major       D = A * Bmn[128(k),128(n)]
 *   mode 2: A in registers (bf16x2 fragments), B MN-major D = A * Bmn
 * A, B bf16 [128,128] row-major; D f32 [128,128].
 * ------------------------------------------------------------------------------------------- */
int yb_umma_probe(const void* A, const void* B, void* D, int mode, void* stream);  /* modes >= 3: A rows shifted by (mode - 2) */

#ifdef __cplusplus
}
#endif
#endif /* YUME_B200_H_ */
