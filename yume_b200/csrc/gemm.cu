// gemm.cu — persistent, warp-specialised wgmma GEMM for sm_90a (H100) with fused epilogues.
//
//   out[M,N] = epilogue( A[M,K] (bf16, row-major) x B[N,K]^T (bf16, row-major, i.e. nn.Linear.weight) + bias[N] )
//
// This is the H100-native replacement for every nn.Linear on the reference's denoise path
// (reference: wan23/modules/model.py:171-174 q/k/v/o, :265-267 ffn, :455-457 text_embedding;
//  wan/modules/model.py:282-287, 358-361, 436-438), with the elementwise work the reference runs as
// separate eager kernels folded into the epilogue:
//   YB_EPI_BF16       out_bf16 = acc + bias                        (q/k/v projections)
//   YB_EPI_GELU_BF16  out_bf16 = gelu_tanh(acc + bias)             (ffn.0 + nn.GELU(approximate='tanh'))
//   YB_EPI_F32        out_f32  = acc + bias                        (patch embedding -> fp32 residual stream)
//   YB_EPI_GELU_ERF_BF16 out_bf16 = gelu_erf(acc + bias)         (MLPProj nn.GELU(), wan/modules/model.py:536)
//   YB_EPI_GATE_RES   resid_f32 += (acc + bias) * gate[tok[m], n]  (o-proj / ffn.2 + adaLN gate + residual add:
//                                                                   model.py:304, 308, 312)
//
// Structure (one CTA per SM, 384 threads = 3 warpgroups):
//   warpgroup 0     TMA producer (one thread): A tile 128x64 and B tile block_n x 64 (128B-swizzled) into an smem ring
//   warpgroups 1-2  consumers: wgmma m64nNk16 over rows [64*(wg-1), +64) of the tile, fp32 accumulators in registers,
//                   then the fused epilogue, in one of two forms chosen by the launch's output layout:
//                   - TMA (1-CTA kernel, plain [M, N] output with a 16-byte row pitch: every yb_gemm_bf16 launch except
//                     RES_BF16 and the N-split layout): each warpgroup writes 64-row x 128-byte boxes of its finished values
//                     into a swizzled staging buffer and one thread hands each box to the TMA unit as an asynchronous store
//                     (GATE_RES: a bulk reduce-add into the fp32 residual stream, done in L2), so the next tile's MMAs start
//                     while the boxes drain;
//                   - registers -> per-warp smem transpose -> full row segments to global (the SM-pair kernel, the conv
//                     modes with their scattered voxel rows, the Ulysses layouts, RES_BF16)
// The SM-pair form (CLUSTER = 2) is a cluster of two CTAs that owns a 256 x block_n tile: each CTA loads its own 128 rows of A
// and HALF of the B tile, and multicasts that half into both CTAs, so the B operand crosses L2 once per pair of SMs.
#include "yb_host.h"
#include "../../include/yume_b200_stream.h"
#include "../../include/yume_b200_vae_rows.h"
#include "../../include/yume_b200_vae_rows_enc.h"
#include "yb_ptx.cuh"

namespace yb {

constexpr int GEMM_BLOCK_M = 128;
constexpr int GEMM_BLOCK_K = 64;  // 64 bf16 = 128 B = one swizzle row
constexpr int GEMM_THREADS = 384;
constexpr int GEMM_MAX_STAGES = 8;
constexpr int GEMM_SMEM_BYTES = 227 * 1024;                 // the H100 per-block maximum
constexpr int GEMM_A_BYTES = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;
constexpr int GEMM_EPI_STAGE_BYTES = 8 * 16 * 36 * 4;       // register epilogue: 8 consumer warps x 16 rows x 36 floats
constexpr int GEMM_EPI_BOX_BYTES = 64 * 128;                // TMA epilogue: one 64-row x 128-byte box (64 bf16 / 32 fp32 columns)
constexpr int GEMM_EPI_TMA_BYTES = 2 * 2 * GEMM_EPI_BOX_BYTES;   // two staging boxes per consumer warpgroup

struct GemmParams {
  int M, N, K;
  const float* bias;      // [N] or null
  void* out;              // bf16 / f32 output, or fp32 residual stream for GATE_RES
  long long ldo;          // row stride of out (elements)
  const float* gate;      // GATE_RES: [U, gate_ld] fp32 table (null => gate = 1)
  long long gate_ld;      // row stride of the gate table
  const int* tok_idx;     // GATE_RES: [M] token -> row of gate table (null => row 0)
  int a_split;            // columns of A per chunk (== K for an ordinary matrix)
  int n_split;            // bf16 outputs: >0 => column block j (width n_split) is written at out + j*split_stride
  long long split_stride;
  const __nv_bfloat16* res;  // YB_EPI_RES_BF16: residual added before the bf16 store, indexed like `out`
  long long res_ld;
  // implicit-GEMM causal conv3d (conv != 0): A rows are output voxels, K = 27 taps x cin_chunks x 64 channels,
  // loaded as 4-D TMA boxes {64, TW, TH, TT} from the replicate-padded channels-last input [T+2, H+2, W+2, Cp]
  int conv, cin_chunks;
  int TW, TH, TT, tiles_w, tiles_h;
  int cT, cH, cW;
  int kh, kw;                   // spatial taps (tap = (dt*kh + dh)*kw + dw)
  int off_t, off_h, off_w;      // subtracted from the box coordinates: 0 when the padding is materialised in the input,
                                // (kt-1, kh/2, kw/2) when it is TMA out-of-bounds zero fill on the unpadded input
  int out_t_mul, out_t_add;     // output frame of input frame t = t*out_t_mul + out_t_add (time_conv interleave)
  int st_t, st_h, st_w;         // conv stride per axis (1 or 2): the tensor map samples every st-th voxel (elementStrides), so a box
                                // still lands as 128 dense rows; cT/cH/cW are OUTPUT extents, the tile origin scales by the stride
  int num_m_tiles, num_n_tiles;
  int block_n, stages;          // N tile (multiple of 32, <= 256) and smem ring depth
  // Tail split-K of the SM-pair kernel (GATE_RES launches): work items [0, sk_full) are whole tiles; item sk_full + u is K segment
  // u % sk_ns (sk_per 64-column blocks) of tile sk_full + u / sk_ns and leaves its raw fp32 accumulator in sk_ws[u][256][block_n]
  // for gemm_splitk_combine_kernel. sk_ns == 1: no split (sk_full == number of tiles).
  int sk_full, sk_ns, sk_per;
  float* sk_ws;
  int tma_out;                  // 1: the epilogue stores through the output tensor map (gemm_has_tma_epilogue instances only)
  // YB_EPI_SP_QKV (internal): the fused q|k|v projection of a Ulysses rank whose epilogue IS the all-to-all — column
  // (part, head h, d) of local token t is stored into the receive buffer of the rank that owns head h (NVLink peer pointer),
  // layout [P(src), Lp, q|k|v of heads/P]; and the per-row sums of squares of the q and k parts (WanRMSNorm spans all heads)
  // are accumulated into sp_sums [Lp][2] for the receiver-side normalisation
  __nv_bfloat16* sp_peers[8];
  float* sp_sums;
  int sp_rank, sp_Lp, sp_Wh, sp_C;
};
constexpr int YB_EPI_SP_QKV = 6;   // not part of the public enum: reached through yb_gemm_sp_qkv only

// CONVW = 1: kw-fused implicit-GEMM conv. The three kw taps of one (dt, dh, channel-chunk) group read the SAME TMA halo
// box of 130 voxels along W; tap dw is fed to the MMA by moving the A descriptor's start address by dw 128-byte rows
// inside the swizzled slab (the swizzle is a function of the absolute smem address, so whole-row shifts stay
// consistent with what TMA wrote — probe modes >= 3). A and B then live in separate rings: one A slab per group, one B
// tile per tap. Cuts the A operand's L2 -> smem traffic 3x, which is what bounds the narrow (<= 128 channel) convs.
constexpr int CONVW_ROWS = GEMM_BLOCK_M + 2;
constexpr int CONVW_A_SLAB = 17 * 1024;  // 130 rows x 128 B = 16640 B, padded to the 1024-B swizzle pattern
constexpr int CONVW_A_STAGES = 4;

// smem: [stages x (A tile | B tile)] [CONVW A ring] [epilogue transpose buffers] [barriers]. The B tile is allocated in whole
// 64-row slabs (the N = 64 MMAs of an odd block_n read the rows past block_n; their columns are never stored).
__host__ __device__ constexpr int gemm_b_bytes(int block_n) { return ((block_n + 63) / 64) * 64 * GEMM_BLOCK_K * 2; }
__host__ __device__ constexpr int gemm_stage_bytes(int block_n, int convw) { return (convw ? 0 : GEMM_A_BYTES) + gemm_b_bytes(block_n); }
__host__ __device__ constexpr int gemm_a_ring_bytes(int convw) { return convw ? CONVW_A_STAGES * CONVW_A_SLAB : 0; }
// instances that carry the TMA epilogue (the launch still picks it per call through p.tma_out), and their epilogue area: the
// larger TMA staging area leaves the 256- / 128-wide rings at 4 / 6 stages; the others keep the transpose buffer only
__host__ __device__ constexpr bool gemm_has_tma_epilogue(int epi, int convw, int cluster) {
  return cluster == 1 && !convw && (epi == YB_EPI_BF16 || epi == YB_EPI_GELU_BF16 || epi == YB_EPI_GELU_ERF_BF16 ||
                                    epi == YB_EPI_F32 || epi == YB_EPI_GATE_RES);
}
// Of those, GELU / GELU_ERF / GATE_RES only ever write a plain matrix (the conv modes and the N-split layout come with BF16 / F32),
// so their 1-CTA instances carry no register epilogue at all.
__host__ __device__ constexpr bool gemm_tma_epilogue_only(int epi, int convw, int cluster) {
  return gemm_has_tma_epilogue(epi, convw, cluster) && epi != YB_EPI_BF16 && epi != YB_EPI_F32;
}
__host__ __device__ constexpr int gemm_epi_bytes(bool tma) { return tma ? GEMM_EPI_TMA_BYTES : GEMM_EPI_STAGE_BYTES; }
static int gemm_stages(int block_n, int convw, int epi_bytes) {
  const int s = (GEMM_SMEM_BYTES - 1024 - 256 - epi_bytes - gemm_a_ring_bytes(convw)) / gemm_stage_bytes(block_n, convw);
  return s > GEMM_MAX_STAGES ? GEMM_MAX_STAGES : s;
}

// One 32-column chunk of the 16 tile rows of a consumer warp, already transposed into `stage` (row pitch 36 floats) by the
// caller. Lane l (< 16) holds my_row / my_tok = logical output row and gate-table row of the warp's tile row l (-1 = none).
// Every global access is a full 64/128-byte row segment shared by 4/8 adjacent lanes.
template <int EPI>
__device__ __forceinline__ void epilogue_rows16(const GemmParams& p, int col0, int my_row, int my_tok, const float* stage, int lane,
                                                float* sq) {
  constexpr bool kBf16Out = (EPI == YB_EPI_BF16 || EPI == YB_EPI_GELU_BF16 || EPI == YB_EPI_GELU_ERF_BF16 ||
                             EPI == YB_EPI_RES_BF16 || EPI == YB_EPI_SP_QKV);
  if (col0 >= p.N) return;
  if (kBf16Out) {
    const int cq = (lane & 3) * 8;  // this lane's 8 columns of the 32-column chunk
    float b[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (p.bias) {
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + cq));
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + cq + 4));
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
    }
    // optional N-split output (Ulysses layout): column block j of width n_split goes to out + j*split_stride
    long long col_off = col0 + cq;
    if (p.n_split > 0) col_off = static_cast<long long>(col0 / p.n_split) * p.split_stride + (col0 % p.n_split) + cq;
    __nv_bfloat16* obase = reinterpret_cast<__nv_bfloat16*>(p.out) + col_off;
    long long ld = p.ldo;
    if (EPI == YB_EPI_SP_QKV) {   // destination = the owner rank's receive buffer; rows are (this rank, local token)
      const int part = col0 / p.sp_C, cin = col0 - part * p.sp_C;
      const int peer = cin / p.sp_Wh;
      ld = 3LL * p.sp_Wh;
      obase = p.sp_peers[peer] + static_cast<long long>(p.sp_rank) * p.sp_Lp * ld + part * p.sp_Wh + (cin - peer * p.sp_Wh) + cq;
    }
    uint4 resv[2];
    if (EPI == YB_EPI_RES_BF16) {  // residual loads first (they may alias the stores for all the compiler knows)
#pragma unroll
      for (int it = 0; it < 2; ++it) {
        const int rowi = __shfl_sync(0xffffffffu, my_row, it * 8 + (lane >> 2));
        resv[it] = make_uint4(0u, 0u, 0u, 0u);
        if (rowi >= 0) resv[it] = *reinterpret_cast<const uint4*>(p.res + static_cast<long long>(rowi) * p.res_ld + col0 + cq);
      }
    }
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int rr = it * 8 + (lane >> 2);
      const int rowi = __shfl_sync(0xffffffffu, my_row, rr);
      const float4 a0 = *reinterpret_cast<const float4*>(stage + rr * 36 + cq);
      const float4 a1 = *reinterpret_cast<const float4*>(stage + rr * 36 + cq + 4);
      float v[8] = {a0.x + b[0], a0.y + b[1], a0.z + b[2], a0.w + b[3], a1.x + b[4], a1.y + b[5], a1.z + b[6], a1.w + b[7]};
      if (EPI == YB_EPI_GELU_BF16) {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = gelu_tanh(v[i]);
      }
      if (EPI == YB_EPI_GELU_ERF_BF16) {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = 0.5f * v[i] * (1.0f + erff(v[i] * 0.7071067811865476f));
      }
      if (EPI == YB_EPI_RES_BF16) {
        const __nv_bfloat162* rh = reinterpret_cast<const __nv_bfloat162*>(&resv[it]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = __bfloat1622float2(rh[i]);
          v[2 * i] += f.x;
          v[2 * i + 1] += f.y;
        }
      }
      if (rowi >= 0) {
        uint4 w;
        w.x = pack_bf16x2(v[0], v[1]);
        w.y = pack_bf16x2(v[2], v[3]);
        w.z = pack_bf16x2(v[4], v[5]);
        w.w = pack_bf16x2(v[6], v[7]);
        *reinterpret_cast<uint4*>(obase + static_cast<long long>(rowi) * ld) = w;
        if (EPI == YB_EPI_SP_QKV) {   // sum of squares of the ROUNDED values (what the receiver normalises)
          const __nv_bfloat162* wh = reinterpret_cast<const __nv_bfloat162*>(&w);
          float acc = 0.f;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = __bfloat1622float2(wh[i]);
            acc += f.x * f.x + f.y * f.y;
          }
          sq[it] += acc;
        }
      }
    }
  } else {
    const int cq = (lane & 7) * 4;  // this lane's 4 columns
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.bias) b = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + cq));
    float* obase = reinterpret_cast<float*>(p.out) + col0 + cq;
    // all loads first, then all stores: the residual rows may alias as far as the compiler can tell, so a
    // load placed after a store would serialise one L2 round trip per row
    float4 xv[4], gv[4];
    int rowv[4];
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int rr = it * 4 + (lane >> 3);
      const int tok = __shfl_sync(0xffffffffu, my_tok, rr);
      rowv[it] = __shfl_sync(0xffffffffu, my_row, rr);
      xv[it] = make_float4(0.f, 0.f, 0.f, 0.f);
      gv[it] = make_float4(1.f, 1.f, 1.f, 1.f);
      if (EPI == YB_EPI_GATE_RES && rowv[it] >= 0) {
        xv[it] = *reinterpret_cast<const float4*>(obase + static_cast<long long>(rowv[it]) * p.ldo);
        if (p.gate) gv[it] = __ldg(reinterpret_cast<const float4*>(p.gate + static_cast<long long>(tok) * p.gate_ld + col0 + cq));
      }
    }
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int rr = it * 4 + (lane >> 3);
      float4 a = *reinterpret_cast<const float4*>(stage + rr * 36 + cq);
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
      if (rowv[it] >= 0) {
        float4* o4 = reinterpret_cast<float4*>(obase + static_cast<long long>(rowv[it]) * p.ldo);
        if (EPI == YB_EPI_F32) {
          *o4 = a;
        } else {  // YB_EPI_GATE_RES
          float4 x = xv[it];
          x.x += a.x * gv[it].x; x.y += a.y * gv[it].y; x.z += a.z * gv[it].z; x.w += a.w * gv[it].w;
          *o4 = x;
        }
      }
    }
  }
}

// TMA epilogue of one consumer warpgroup: its 64 x NM accumulator (rows row0.., columns col0..) leaves as boxes of 64 rows x
// 128 bytes, 64 bf16 or 32 fp32 columns each. Per box every thread finishes its values in registers (bias, GELU, bf16 rounding;
// GATE_RES: (acc + bias) * gate[tok[row], col]) and writes them into a staging buffer in the output tensor map's 128B swizzle
// (16-byte chunk c of box row r at chunk c ^ (r & 7)); one thread then issues the box as a TMA store, or as a bulk reduce-add
// into the fp32 residual for GATE_RES, and commits it as a bulk group. Two buffers alternate: a buffer is rewritten only after
// the group that read it two boxes ago has finished reading (wait_group.read 1). `nbox` counts this warpgroup's boxes across
// tiles so the alternation carries on. Rows past M and columns past N are clipped by the TMA unit.
template <int EPI, int NM>
__device__ __forceinline__ void epilogue_tma(const GemmParams& p, const CUtensorMap* tmO, const float (&acc)[128], uint8_t* bufs,
                                             int row0, int col0, int wg, int wtid, uint32_t& nbox) {
  constexpr bool kF32 = (EPI == YB_EPI_F32 || EPI == YB_EPI_GATE_RES);
  constexpr int BOX_COLS = kF32 ? 32 : 64;
  constexpr int GROUPS = BOX_COLS / 8;   // accumulator column groups of 8 per box
  if (row0 >= p.M) return;               // uniform over the warpgroup
  const int lane = wtid & 31;
  const int r = (wtid >> 5) * 16 + (lane >> 2);   // this thread's box rows r and r + 8 (fragment rows); (r & 7) == lane >> 2
  const int sw = lane >> 2, c2 = 2 * (lane & 3);
  const int ncols = min(NM, p.N - col0);
  const float* g_lo = nullptr;
  const float* g_hi = nullptr;
  if (EPI == YB_EPI_GATE_RES && p.gate != nullptr) {
    int t_lo = 0, t_hi = 0;
    if (p.tok_idx != nullptr) {
      if (row0 + r < p.M) t_lo = p.tok_idx[row0 + r];
      if (row0 + r + 8 < p.M) t_hi = p.tok_idx[row0 + r + 8];
    }
    g_lo = p.gate + static_cast<long long>(t_lo) * p.gate_ld;
    g_hi = p.gate + static_cast<long long>(t_hi) * p.gate_ld;
  }
#pragma unroll
  for (int s = 0; s < NM / BOX_COLS; ++s) {
    if (s * BOX_COLS < ncols) {
      uint8_t* buf = bufs + (nbox & 1) * GEMM_EPI_BOX_BYTES;
      if (wtid == 0) bulk_wait_read<1>();   // the store that last read this buffer is done with it
      named_bar_sync(1 + wg, 128);
      // one group of 8 columns at a time (the accumulator of the later boxes is still live): finished values of rows r / r + 8,
      // columns s * BOX_COLS + 8j + c2, +1
#pragma unroll
      for (int j = 0; j < GROUPS; ++j) {
        const int g = s * GROUPS + j;
        const int col = col0 + s * BOX_COLS + 8 * j + c2;
        float2 b = make_float2(0.f, 0.f);
        const bool in = s * BOX_COLS + 8 * j < ncols;   // N % 32 == 0: a group of 8 columns is all in or all out
        if (p.bias && in) b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
        float2 lo = make_float2(acc[4 * g] + b.x, acc[4 * g + 1] + b.y);
        float2 hi = make_float2(acc[4 * g + 2] + b.x, acc[4 * g + 3] + b.y);
        if (EPI == YB_EPI_GELU_BF16) {
          lo = make_float2(gelu_tanh(lo.x), gelu_tanh(lo.y));
          hi = make_float2(gelu_tanh(hi.x), gelu_tanh(hi.y));
        }
        if (EPI == YB_EPI_GELU_ERF_BF16) {
          auto ge = [](float v) { return 0.5f * v * (1.0f + erff(v * 0.7071067811865476f)); };
          lo = make_float2(ge(lo.x), ge(lo.y));
          hi = make_float2(ge(hi.x), ge(hi.y));
        }
        if (EPI == YB_EPI_GATE_RES && g_lo != nullptr && in) {
          const float2 gl = __ldg(reinterpret_cast<const float2*>(g_lo + col));
          const float2 gh = __ldg(reinterpret_cast<const float2*>(g_hi + col));
          lo = make_float2(lo.x * gl.x, lo.y * gl.y);
          hi = make_float2(hi.x * gh.x, hi.y * gh.y);
        }
        if (kF32) {   // 32 bytes per group: chunks 2j, 2j + 1; this pair at byte 8 * (lane & 1) of chunk 2j + (lane & 3) / 2
          const int off = (((2 * j + ((lane & 3) >> 1)) ^ sw) << 4) + 8 * (lane & 1);
          *reinterpret_cast<float2*>(buf + r * 128 + off) = lo;
          *reinterpret_cast<float2*>(buf + (r + 8) * 128 + off) = hi;
        } else {      // 16 bytes per group: chunk j; this pair at byte 4 * (lane & 3)
          const int off = ((j ^ sw) << 4) + 4 * (lane & 3);
          *reinterpret_cast<uint32_t*>(buf + r * 128 + off) = pack_bf16x2(lo.x, lo.y);
          *reinterpret_cast<uint32_t*>(buf + (r + 8) * 128 + off) = pack_bf16x2(hi.x, hi.y);
        }
      }
      fence_proxy_async_smem();   // make the generic-proxy writes visible to the TMA unit
      named_bar_sync(1 + wg, 128);
      if (wtid == 0) {
        if (EPI == YB_EPI_GATE_RES) tma_reduce_add_2d(tmO, buf, col0 + s * BOX_COLS, row0);
        else tma_store_2d(tmO, buf, col0 + s * BOX_COLS, row0);
        bulk_commit();
      }
      ++nbox;
    }
  }
}

// one 64-wide K block of this warpgroup's 64 x block_n accumulator: 4 k-steps of 16 (32 B inside the 128-B swizzle row).
// NM = MMA width: 256 / 128 (block_n equal to it) or 64 (any multiple of 32: block_n / 64 rounded up N = 64 MMAs). A compile-time
// choice: with the three forms in one kernel ptxas serialises the wgmma pipeline.
template <int NM>
__device__ __forceinline__ void gemm_mma_k64(float (&acc)[128], uint32_t sa, uint32_t sb, int block_n, bool zero_first) {
  const uint64_t ad0 = make_smem_desc_sw128(sa, 16, 1024), bd0 = make_smem_desc_sw128(sb, 16, 1024);
  const int nb64 = (block_n + 63) >> 6;
#pragma unroll
  for (int k = 0; k < GEMM_BLOCK_K / 16; ++k) {
    const uint64_t ad = ad0 + 2 * k, bd = bd0 + 2 * k;
    const uint32_t accum = (zero_first && k == 0) ? 0u : 1u;
    if (NM == 256) {
      wgmma_ss_n256<0>(acc, ad, bd, accum);
    } else if (NM == 128) {
      wgmma_ss_n128<0>(acc, ad, bd, accum);
    } else {   // 64-column slabs of the B tile sit 8 KB apart
      wgmma_ss_n64<0>(acc, ad, bd, accum);
      if (nb64 > 1) wgmma_ss_n64<32>(acc, ad, bd + (8192 >> 4), accum);
      if (nb64 > 2) wgmma_ss_n64<64>(acc, ad, bd + (16384 >> 4), accum);
      if (nb64 > 3) wgmma_ss_n64<96>(acc, ad, bd + (24576 >> 4), accum);
    }
  }
}

template <int CLUSTER>
__device__ __forceinline__ void release_slot(uint64_t* bar, int lane) {
  __syncwarp();
  if (lane == 0) {
    if (CLUSTER == 1) {
      mbar_arrive(bar);
    } else {   // the slot is refilled by BOTH CTAs' multicasts: free it in both
      mbar_arrive_cluster(bar, 0);
      mbar_arrive_cluster(bar, 1);
    }
  }
}

template <int EPI, int CONVW, int CLUSTER, int NM>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO,
            const GemmParams p) {
  static_assert(!(CONVW && CLUSTER != 1), "the kw-fused conv runs on single CTAs");
  constexpr bool kTmaEpi = gemm_has_tma_epilogue(EPI, CONVW, CLUSTER);
  const bool tma_out = gemm_tma_epilogue_only(EPI, CONVW, CLUSTER) || (kTmaEpi && p.tma_out);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int block_n = p.block_n, stages = p.stages;
  const int stage_bytes = gemm_stage_bytes(block_n, CONVW);
  uint8_t* a_ring = smem + stages * stage_bytes;
  float* epi = reinterpret_cast<float*>(a_ring + gemm_a_ring_bytes(CONVW));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(epi) + gemm_epi_bytes(kTmaEpi));
  uint64_t* empty_bar = full_bar + GEMM_MAX_STAGES;
  uint64_t* a_full = empty_bar + GEMM_MAX_STAGES;   // CONVW only
  uint64_t* a_empty = a_full + CONVW_A_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = CLUSTER == 2 ? static_cast<int>(cluster_ctarank()) : 0;
  const int tile_first = blockIdx.x / CLUSTER, tile_step = gridDim.x / CLUSTER;
  const int num_tiles = p.num_m_tiles * p.num_n_tiles;   // tiles of (128 * CLUSTER) x block_n
  const int num_kb = (p.K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;
  const int num_work = p.sk_full + (num_tiles - p.sk_full) * p.sk_ns;   // == num_tiles without a split tail
  // work item -> (tile, K-block range, partial slot or -1); every role walks the same sequence
  auto decode_work = [&](int w, int& tile, int& kb0, int& kb1, int& part) {
    tile = w; kb0 = 0; kb1 = num_kb; part = -1;
    if (w >= p.sk_full) {
      const int u = w - p.sk_full;
      tile = p.sk_full + u / p.sk_ns;
      kb0 = (u % p.sk_ns) * p.sk_per;
      kb1 = min(num_kb, kb0 + p.sk_per);
      part = u;
    }
  };
  // conv tile -> origin of its TT x TH x TW output box
  auto conv_box = [&](int mt, int& it, int& ih, int& iw) {
    const int per_t = p.tiles_h * p.tiles_w;
    it = mt / per_t;
    const int rem = mt - it * per_t;
    ih = rem / p.tiles_w;
    iw = rem - ih * p.tiles_w;
  };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (tma_out) tma_prefetch_desc(&tmO);
    for (int i = 0; i < stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8 * CLUSTER);   // every consumer warp of every CTA that writes into the slot
    }
    for (int i = 0; i < (CONVW ? CONVW_A_STAGES : 0); ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (CLUSTER > 1) cluster_sync_all();   // every barrier of the pair exists before any remote signal

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      // ------------------------------- TMA producer -------------------------------
      int stage = 0, a_stage = 0;
      uint32_t phase = 0, a_phase = 0;
      for (int w = tile_first; w < num_work; w += tile_step) {
        int tile, kb0, kb1, part, m_tile, n_tile;
        decode_work(w, tile, kb0, kb1, part);
        tile_coords(tile, p.num_m_tiles, p.num_n_tiles, m_tile, n_tile);
        if (CONVW) {
          int it, ih, iw;
          conv_box(m_tile, it, ih, iw);
          const int groups = num_kb / 3;   // (dt, dh, channel chunk)
          for (int g = 0; g < groups; ++g) {
            const int tdh = g / p.cin_chunks, cc = g - tdh * p.cin_chunks;
            const int dt = tdh / p.kh, dh = tdh - dt * p.kh;
            mbar_wait(&a_empty[a_stage], a_phase ^ 1);
            mbar_arrive_expect_tx(&a_full[a_stage], CONVW_ROWS * GEMM_BLOCK_K * 2);
            tma_load_4d(a_ring + a_stage * CONVW_A_SLAB, &tmA, &a_full[a_stage], cc * GEMM_BLOCK_K, iw * GEMM_BLOCK_M - p.off_w,
                        ih + dh - p.off_h, it + dt - p.off_t);
            if (++a_stage == CONVW_A_STAGES) {
              a_stage = 0;
              a_phase ^= 1;
            }
#pragma unroll 1
            for (int dw = 0; dw < 3; ++dw) {
              mbar_wait(&empty_bar[stage], phase ^ 1);
              mbar_arrive_expect_tx(&full_bar[stage], block_n * GEMM_BLOCK_K * 2);
              tma_load_2d(smem + stage * stage_bytes, &tmB, &full_bar[stage], ((tdh * 3 + dw) * p.cin_chunks + cc) * GEMM_BLOCK_K,
                          n_tile * block_n);
              if (++stage == stages) {
                stage = 0;
                phase ^= 1;
              }
            }
          }
          continue;
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          if (CLUSTER > 1) mbar_wait_cluster(&empty_bar[stage], phase ^ 1);
          else mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * stage_bytes;
          uint8_t* sb = sa + GEMM_A_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], GEMM_A_BYTES + block_n * GEMM_BLOCK_K * 2);
          const int kcol = kb * GEMM_BLOCK_K;
          const int mt = m_tile * CLUSTER + rank;   // this CTA's 128-row block (a pair's second block past the end is all zeros)
          if (p.conv) {
            // tap (dt, dh, dw) reads padded voxel (t + dt, h + dh, w + dw): P[tp][hp][wp] = X[max(tp-2,0)][clamp(hp-1)]
            // [clamp(wp-1)] — temporal pad 2 in front only (causal), replicate everywhere
            const int tap = kb / p.cin_chunks, cc = kb - tap * p.cin_chunks;
            const int dt = tap / (p.kh * p.kw), dh = (tap / p.kw) % p.kh, dw = tap % p.kw;
            int it, ih, iw;
            conv_box(mt, it, ih, iw);
            tma_load_4d(sa, &tmA, &full_bar[stage], cc * GEMM_BLOCK_K, iw * p.TW * p.st_w + dw - p.off_w,
                        ih * p.TH * p.st_h + dh - p.off_h, it * p.TT * p.st_t + dt - p.off_t);
          } else {
            // A goes through a 3-D map [chunk, row, col]: logical column k lives in chunk k / a_split (one chunk when
            // the operand is an ordinary matrix; P chunks for the Ulysses-received attention output)
            const int chunk = kcol / p.a_split;
            tma_load_3d(sa, &tmA, &full_bar[stage], kcol - chunk * p.a_split, mt * GEMM_BLOCK_M, chunk);
          }
          if (CLUSTER == 1) {
            tma_load_2d(sb, &tmB, &full_bar[stage], kcol, n_tile * block_n);
          } else {
            const int half = block_n / 2;
            tma_load_2d_multicast(sb + rank * half * GEMM_BLOCK_K * 2, &tmB, &full_bar[stage], kcol, n_tile * block_n + rank * half,
                                  static_cast<uint16_t>(3));
          }
          if (++stage == stages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ------------------------------- consumers: MMA + epilogue -------------------------------
    setmaxnreg_inc<232>();   // 128 x 40 + 256 x 232 <= 65536
    const int wg = (warp >> 2) - 1;   // rows [64 * wg, +64) of the CTA's 128-row tile
    const int r0 = wg * 64 + (warp & 3) * 16;   // first of the 16 tile rows this warp stores
    float* stage_buf = epi + (warp - 4) * (16 * 36);
    uint8_t* box_bufs = reinterpret_cast<uint8_t*>(epi) + wg * 2 * GEMM_EPI_BOX_BYTES;   // TMA epilogue: this warpgroup's two boxes
    uint32_t nbox = 0;
    int stage = 0, a_stage = 0;
    uint32_t phase = 0, a_phase = 0;
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    for (int w = tile_first; w < num_work; w += tile_step) {
      int tile, kb0, kb1, part, m_tile, n_tile;
      decode_work(w, tile, kb0, kb1, part);
      tile_coords(tile, p.num_m_tiles, p.num_n_tiles, m_tile, n_tile);
      const int mt = m_tile * CLUSTER + rank;
      // register epilogue: logical output row of tile row r0 + (lane & 15), the matrix row or the voxel index of a conv tile;
      // -1 = none
      int my_row = -1;
      if (!tma_out) {
        const int r = r0 + (lane & 15);
        if (p.conv) {
          int it, ih, iw;
          conv_box(mt, it, ih, iw);
          const int tw = r % p.TW, th = (r / p.TW) % p.TH, tt = r / (p.TW * p.TH);
          const int t = it * p.TT + tt, h = ih * p.TH + th, ww = iw * p.TW + tw;
          my_row = (t < p.cT && h < p.cH && ww < p.cW) ? ((t * p.out_t_mul + p.out_t_add) * p.cH + h) * p.cW + ww : -1;
        } else {
          const int row = mt * GEMM_BLOCK_M + r;
          my_row = row < p.M ? row : -1;
        }
      }
      if (EPI == YB_EPI_GATE_RES && part < 0 && my_row >= 0 && lane < 16) {
        // the residual rows of this tile are cold in HBM: pull them into L2 while the accumulator is computed
        const char* xrow = reinterpret_cast<const char*>(reinterpret_cast<const float*>(p.out) +
                                                         static_cast<long long>(my_row) * p.ldo + n_tile * block_n);
        const int ncols = min(block_n, p.N - n_tile * block_n);
        for (int b = 0; b < ncols * 4; b += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(xrow + b));
      }
      // main loop: wgmma groups of one stage stay in flight while the next stage is issued; a slot is released once the
      // MMAs that read it have completed
      int prev = -1;
      if (CONVW) {
        int prev_a = -1;
        const int groups = num_kb / 3;
        for (int g = 0; g < groups; ++g) {
          mbar_wait(&a_full[a_stage], a_phase);
          const uint32_t sa = smem_u32(a_ring + a_stage * CONVW_A_SLAB) + wg * 64 * 128;
#pragma unroll 1
          for (int dw = 0; dw < 3; ++dw) {
            mbar_wait(&full_bar[stage], phase);
            fence_regs(acc);
            wgmma_fence();
            gemm_mma_k64<NM>(acc, sa + dw * 128, smem_u32(smem + stage * stage_bytes), block_n, g == 0 && dw == 0);   // tap dw = rows [dw, dw + 128)
            wgmma_commit();
            wgmma_wait<1>();
            fence_regs(acc);
            if (prev >= 0) release_slot<1>(&empty_bar[prev], lane);
            if (dw == 0 && prev_a >= 0) {
              release_slot<1>(&a_empty[prev_a], lane);
              prev_a = -1;
            }
            prev = stage;
            if (++stage == stages) {
              stage = 0;
              phase ^= 1;
            }
          }
          prev_a = a_stage;
          if (++a_stage == CONVW_A_STAGES) {
            a_stage = 0;
            a_phase ^= 1;
          }
        }
        wgmma_wait<0>();
        fence_regs(acc);
        if (prev >= 0) release_slot<1>(&empty_bar[prev], lane);
        if (prev_a >= 0) release_slot<1>(&a_empty[prev_a], lane);
      } else {
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_u32(smem + stage * stage_bytes);
          fence_regs(acc);
          wgmma_fence();
          gemm_mma_k64<NM>(acc, sa + wg * 64 * 128, sa + GEMM_A_BYTES, block_n, kb == kb0);
          wgmma_commit();
          wgmma_wait<1>();
          fence_regs(acc);
          if (prev >= 0) release_slot<CLUSTER>(&empty_bar[prev], lane);
          prev = stage;
          if (++stage == stages) {
            stage = 0;
            phase ^= 1;
          }
        }
        wgmma_wait<0>();
        fence_regs(acc);
        if (prev >= 0) release_slot<CLUSTER>(&empty_bar[prev], lane);
      }

      const int q4 = lane >> 2, c2 = 2 * (lane & 3);   // fragment: rows q4 / q4 + 8, columns 8g + c2, +1
      if (part >= 0) {
        // K segment of a split tail tile: the raw fp32 accumulator goes to the workspace, row-major [256][block_n]; the fused
        // epilogue runs in gemm_splitk_combine_kernel over the sum of the segments
        float* wbase = p.sk_ws + (static_cast<long long>(part) * 256 + rank * GEMM_BLOCK_M + r0) * block_n;
#pragma unroll
        for (int g = 0; g < 32; ++g) {
          if (g * 8 < block_n) {
            *reinterpret_cast<float2*>(wbase + q4 * block_n + g * 8 + c2) = make_float2(acc[4 * g], acc[4 * g + 1]);
            *reinterpret_cast<float2*>(wbase + (q4 + 8) * block_n + g * 8 + c2) = make_float2(acc[4 * g + 2], acc[4 * g + 3]);
          }
        }
        continue;
      }
      if (tma_out) {
        epilogue_tma<EPI, NM>(p, &tmO, acc, box_bufs, mt * GEMM_BLOCK_M + wg * 64, n_tile * block_n, wg, threadIdx.x & 127, nbox);
        continue;
      }
      int my_tok = 0;  // gate-table row of tile row r0 + lane
      if (EPI == YB_EPI_GATE_RES && p.gate != nullptr && p.tok_idx != nullptr && my_row >= 0) my_tok = p.tok_idx[my_row];
      float sq[2] = {0.f, 0.f};   // SP_QKV: running sum of squares of warp rows it*8 + lane/4 over the current part
      auto flush_sq = [&](int part_) {   // 4 lanes share a row: reduce, one atomic per row and (tile, part)
#pragma unroll
        for (int it = 0; it < 2; ++it) {
          float v = sq[it];
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          const int rowi = __shfl_sync(0xffffffffu, my_row, it * 8 + (lane >> 2));
          if ((lane & 3) == 0 && rowi >= 0 && part_ < 2) atomicAdd(p.sp_sums + rowi * 2 + part_, v);
          sq[it] = 0.f;
        }
      };
      int cur_part = (EPI == YB_EPI_SP_QKV) ? (n_tile * block_n) / p.sp_C : 0;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        if (c * 32 < block_n) {
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            const int i = 4 * (4 * c + g);
            *reinterpret_cast<float2*>(stage_buf + q4 * 36 + g * 8 + c2) = make_float2(acc[i], acc[i + 1]);
            *reinterpret_cast<float2*>(stage_buf + (q4 + 8) * 36 + g * 8 + c2) = make_float2(acc[i + 2], acc[i + 3]);
          }
          __syncwarp();
          const int col0 = n_tile * block_n + c * 32;
          if (EPI == YB_EPI_SP_QKV && col0 < p.N) {
            const int pt = col0 / p.sp_C;
            if (pt != cur_part) {
              flush_sq(cur_part);
              cur_part = pt;
            }
          }
          epilogue_rows16<EPI>(p, col0, my_row, my_tok, stage_buf, lane, sq);
          __syncwarp();
        }
      }
      if (EPI == YB_EPI_SP_QKV) flush_sq(cur_part);
    }
    if (tma_out && (threadIdx.x & 127) == 0) bulk_wait<0>();   // every box written before the CTA (and its smem) goes away
  }
  if (CLUSTER > 1) cluster_sync_all();   // no CTA leaves while its peer may still multicast into it or arrive on its barriers
}

// Fused epilogue of the split tail tiles (YB_EPI_GATE_RES): x[row, col] += (sum of the K-segment partials + bias[col]) * gate[tok, col],
// segments added in index order (deterministic). One thread per 4 columns of one tile row.
__global__ void __launch_bounds__(256) gemm_splitk_combine_kernel(const GemmParams p, int tail_tiles) {
  const int block_n = p.block_n, quads = block_n >> 2;
  const long long total = static_cast<long long>(tail_tiles) * 256 * quads;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cq = static_cast<int>(i % quads) * 4;
    const long long rr = i / quads;
    const int r = static_cast<int>(rr & 255);
    const int t = static_cast<int>(rr >> 8);
    int m_tile, n_tile;
    tile_coords(p.sk_full + t, p.num_m_tiles, p.num_n_tiles, m_tile, n_tile);
    const int row = m_tile * 256 + r, col = n_tile * block_n + cq;
    if (row >= p.M || col >= p.N) continue;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int sg = 0; sg < p.sk_ns; ++sg) {
      const float4 v = *reinterpret_cast<const float4*>(p.sk_ws + ((static_cast<long long>(t) * p.sk_ns + sg) * 256 + r) * block_n + cq);
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
    if (p.bias) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + col));
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    float4 g = make_float4(1.f, 1.f, 1.f, 1.f);
    if (p.gate) {
      const long long tok = p.tok_idx ? p.tok_idx[row] : 0;
      g = __ldg(reinterpret_cast<const float4*>(p.gate + tok * p.gate_ld + col));
    }
    float4* xp = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + static_cast<long long>(row) * p.ldo + col);
    float4 x = *xp;
    x.x += a.x * g.x; x.y += a.y * g.y; x.z += a.z * g.z; x.w += a.w * g.w;
    *xp = x;
  }
}

// Tail split-K plan (host arithmetic, exported through yb_gemm_splitk_plan): `tiles` output tiles on `clusters` SM pairs leave a
// last wave of r = tiles % clusters tiles; cutting each of them into ns K segments costs ceil(r * ns / clusters) sub-waves, each
// 1 / ns of a tile plus a fixed 5 / num_kb of a tile (pipeline fill + fp32 dump of the partial, ~5 K blocks of 64 columns at the
// ~1.8 us an SM pair spends per K block), plus the combine launch (6 / num_kb) and 1 % per segment of workspace traffic.
// Calibrated on one H100 SXM (700 W), x += (A W^T + b) * gate, N = 3072, unsplit -> best split, us: M = 4620, K = 3072
// 349 -> 327 (2 segments); M = 4620, K = 14336 1460 -> 1405 (2); M = 1500, K = 3072 175 -> 117 (6); M = 2310 at K = 3072 and
// 14336 (54 tail tiles: two sub-waves) only lose, 184 -> 201 and 742 -> 785. The model picks each of these.
static void gemm_splitk_plan(int tiles, int num_kb, int clusters, int force_ns, int* full, int* ns, int* per) {
  *full = tiles; *ns = 1; *per = num_kb;
  if (clusters <= 0 || force_ns == 1) return;
  int r = tiles % clusters;
  if (force_ns >= 2) {
    if (num_kb < 2 * force_ns) return;
    if (tiles <= clusters || r == 0) r = tiles < clusters ? tiles : clusters;   // tests: split the last wave whatever its fill
    *ns = force_ns;
  } else {
    if (tiles <= clusters || r == 0) return;
    double best = 0.85;
    for (int n = 2; n <= 12 && num_kb / n >= 8; ++n) {
      const int pr = (num_kb + n - 1) / n;
      const double cost = static_cast<double>((r * n + clusters - 1) / clusters) * (pr + 5.0) / num_kb + 6.0 / num_kb + 0.01 * n;
      if (cost < best) { best = cost; *ns = n; }
    }
    if (*ns == 1) return;
  }
  *per = (num_kb + *ns - 1) / *ns;
  while (*ns > 1 && (*ns - 1) * *per >= num_kb) --*ns;   // every segment owns at least one K block
  if (*ns == 1) { *per = num_kb; return; }
  *full = tiles - r;
}

// N tile of the SM-pair kernel: 256, or N itself rounded up to 32 for narrower outputs. Host arithmetic only — exported through
// yb_gemm_plan.
static int pair_block_n(int M, int N, int clusters) {
  (void)M;
  (void)clusters;
  return N >= 256 ? 256 : ((N + 31) / 32) * 32;
}

// CTA pairs the device holds at once: asked of the driver, SM count / 2 if the query is unavailable
template <typename Kern>
static int pair_max_clusters(Kern kern) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(2 * (sm_count() / 2));
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = GEMM_SMEM_BYTES;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = 2;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess || n <= 0) {
    (void)cudaGetLastError();
    n = sm_count() / 2;
  }
  return n;
}

// p.block_n set by the caller; CLUSTER = 2 is the SM-pair form (256-row tiles, multicast B halves). tmO: the output tensor map
// of the TMA epilogue, or null for the register epilogue.
template <int EPI, int CONVW, int CLUSTER>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap* tmO, GemmParams& p, cudaStream_t stream,
                       int split_k = 1, void* ws = nullptr, long long ws_bytes = 0) {
  static const CUtensorMap no_map = {};
  if (gemm_tma_epilogue_only(EPI, CONVW, CLUSTER) && tmO == nullptr) return YB_ERR_ARG;
  p.tma_out = gemm_has_tma_epilogue(EPI, CONVW, CLUSTER) && tmO != nullptr;
  if (!p.tma_out) tmO = &no_map;
  // MMA width: the 1-CTA kernel runs 128- and 256-wide tiles only
  const int nm = p.block_n == 256 ? 2 : p.block_n == 128 ? 1 : 0;
  if (CLUSTER == 1 && nm == 0) return YB_ERR_ARG;
  auto kern = nm == 2 ? gemm_kernel<EPI, CONVW, CLUSTER, 256> : nm == 1 ? gemm_kernel<EPI, CONVW, CLUSTER, 128>
                      : gemm_kernel<EPI, CONVW, CLUSTER, CLUSTER == 1 ? 128 : 64>;
  static bool attr_set[3][kMaxDevices] = {};
  if (int rc = ensure_dynamic_smem(kern, GEMM_SMEM_BYTES, attr_set[nm], "gemm")) return rc;
  if (CLUSTER == 2) p.num_m_tiles = p.conv ? (p.num_m_tiles + 1) / 2 : (p.M + 255) / 256;   // conv: pairs of 128-voxel boxes
  else if (!p.conv) p.num_m_tiles = (p.M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M;
  p.num_n_tiles = (p.N + p.block_n - 1) / p.block_n;
  p.stages = gemm_stages(p.block_n, CONVW, gemm_epi_bytes(gemm_has_tma_epilogue(EPI, CONVW, CLUSTER)));
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  // persistent grid: one CTA per SM, or the number of CTA pairs the device holds at once (asked of the driver once per device)
  static int max_clusters[kMaxDevices] = {0};
  const int dev = current_device();
  if (max_clusters[dev] == 0) max_clusters[dev] = CLUSTER == 2 ? pair_max_clusters(kern) : sm_count();
  p.sk_full = tiles; p.sk_ns = 1; p.sk_per = 0; p.sk_ws = nullptr;
  int tail = 0;
  if (CLUSTER == 2 && EPI == YB_EPI_GATE_RES && !p.conv && ws != nullptr && split_k != 1) {
    const int num_kb = (p.K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;
    gemm_splitk_plan(tiles, num_kb, max_clusters[dev], split_k, &p.sk_full, &p.sk_ns, &p.sk_per);
    tail = tiles - p.sk_full;
    const long long need = static_cast<long long>(tail) * p.sk_ns * 256 * p.block_n * 4;
    if (tail > 0 && (ws_bytes < need || (reinterpret_cast<uintptr_t>(ws) & 0xF))) {   // workspace too small: unsplit, same result
      p.sk_full = tiles; p.sk_ns = 1; tail = 0;
    }
    if (tail > 0) p.sk_ws = static_cast<float*>(ws);
  }
  const int work = p.sk_full + tail * p.sk_ns;
  const int groups = work < max_clusters[dev] ? work : max_clusters[dev];
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(groups * CLUSTER);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = GEMM_SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = CLUSTER;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  (void)cudaLaunchKernelEx(&cfg, kern, tmA, tmB, *tmO, p);   // a failed launch is reported by check_launch
  int rc = check_launch("gemm");
  if (rc || tail == 0) return rc;
  const long long total = static_cast<long long>(tail) * 256 * (p.block_n / 4);
  gemm_splitk_combine_kernel<<<static_cast<int>((total + 255) / 256), 256, 0, stream>>>(p, tail);
  return check_launch("gemm_splitk_combine");
}

// Tile plan of one conv launch (pure host arithmetic; exported as yb_conv3d_plan for the CPU test-suite).
// The 128-voxel output tile is a TT x TH x TW box (powers of two): pick the shape that wastes the fewest rows on ragged
// edges (W = 80 / 160 / 320 of the 720p Wan2.2 decode would lose 38 / 38 / 17 % with a fixed 128-wide row tile); ties go
// to the widest box (fewest halo re-reads).
// kw-fused mode (one 130-voxel halo box feeds the three kw taps) needs the one-row 128-voxel tile; it is taken when that
// tile shape costs little utilisation — generously for 128-wide N tiles (operand-fetch bound), only when nearly free for
// 256-wide ones (MMA bound). fuse_policy: 0 = auto, 1 = off, 2 = force (tests).
static void conv_plan(int T, int H, int W, int block_n, int kw, int fuse_policy, int* TW, int* TH, int* TT, bool* fused) {
  auto pow2_ge = [](int v) { int p = 1; while (p < v) p <<= 1; return p; };
  double best = -1.0;
  const double vox = static_cast<double>(T) * H * W;
  for (int tw = 128; tw >= 1; tw >>= 1) {
    if (tw > pow2_ge(W)) continue;
    for (int th = 128 / tw; th >= 1; th >>= 1) {
      const int tt = 128 / (tw * th);
      const double tiles = static_cast<double>((W + tw - 1) / tw) * ((H + th - 1) / th) * ((T + tt - 1) / tt);
      const double util = vox / (tiles * 128.0);
      if (util > best + 1e-9) { best = util; *TW = tw; *TH = th; *TT = tt; }
    }
  }
  *fused = false;
  if (kw == 3 && fuse_policy != 1 && (W >= 64 || fuse_policy == 2)) {
    const double util128 = static_cast<double>(W) / (((W + 127) / 128) * 128.0);
    *fused = fuse_policy == 2 || util128 >= (block_n == 128 ? 0.70 : 0.95) * best;
  }
  if (*fused) { *TW = 128; *TH = 1; *TT = 1; }
}

}  // namespace yb

// Fused q|k|v projection + Ulysses all-to-all (see GemmParams): out rows go straight into the owner ranks' receive buffers.
extern "C" int yb_gemm_sp_qkv(const void* A, long long lda, const void* W, const void* bias, int Lp_rows, int C, int K,
                              void* const* peers, int world, int rank, int Lp, void* sums, void* stream_) {
  using namespace yb;
  if (!A || !W || !peers || !sums || Lp_rows <= 0 || C <= 0 || K <= 0) return YB_ERR_ARG;
  if (world < 2 || world > 8 || rank < 0 || rank >= world || Lp < Lp_rows) return YB_ERR_ARG;
  if (C % (world * 128) != 0 || K % 8 != 0 || (lda % 8)) return YB_ERR_SHAPE;
  GemmParams p = {};
  p.M = Lp_rows;
  p.N = 3 * C;
  p.K = K;
  p.bias = static_cast<const float*>(bias);
  p.out = peers[rank];
  p.ldo = 3LL * (C / world);
  p.a_split = K;
  p.sp_rank = rank;
  p.sp_Lp = Lp;
  p.sp_Wh = C / world;
  p.sp_C = C;
  p.sp_sums = static_cast<float*>(sums);
  for (int i = 0; i < 8; ++i) p.sp_peers[i] = i < world ? static_cast<__nv_bfloat16*>(peers[i]) : nullptr;
  p.block_n = pair_block_n(p.M, p.N, sm_count() / 2);
  CUtensorMap tmA, tmB;
  int rc = make_tmap_bf16_3d(&tmA, A, 1, p.M, K, lda, lda * (long long)p.M + 8, GEMM_BLOCK_M, GEMM_BLOCK_K);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmB, W, p.N, K, K, p.block_n / 2, GEMM_BLOCK_K);
  if (rc) return rc;
  return launch_gemm<YB_EPI_SP_QKV, 0, 2>(tmA, tmB, nullptr, p, reinterpret_cast<cudaStream_t>(stream_));
}

// Automatic kernel / tile choice of yb_gemm_bf16: the 1-CTA kernel for every shape. On the H100 (700 W) the SM-pair form measured
// 321-339 TFLOP/s on the three DiT GEMM shapes at L = 18 480 against 624-684 for the 1-CTA kernel, so it runs only when asked for
// (cta_pair = 2) and as the fused Ulysses q|k|v all-to-all (yb_gemm_sp_qkv).
extern "C" int yb_gemm_plan(int M, int N, int sms, int* out4) {
  if (M <= 0 || N <= 0 || sms < 2 || !out4) return YB_ERR_ARG;
  out4[0] = 0;
  out4[1] = (N % 256 == 0 || N > 1024) ? 256 : 128;
  out4[2] = (M + yb::GEMM_BLOCK_M - 1) / yb::GEMM_BLOCK_M;
  out4[3] = (N + out4[1] - 1) / out4[1];
  return YB_OK;
}

extern "C" int yb_conv3d_plan(int T, int H, int W, int Cout, int kw, int fuse_w, int* out4) {
  if (T <= 0 || H <= 0 || W <= 0 || Cout <= 0 || (kw != 1 && kw != 3) || fuse_w < 0 || fuse_w > 2 || !out4) return YB_ERR_ARG;
  bool fused = false;
  yb::conv_plan(T, H, W, (Cout % 256 == 0) ? 256 : 128, kw, fuse_w, &out4[0], &out4[1], &out4[2], &fused);
  out4[3] = fused ? 1 : 0;
  return YB_OK;
}

// Tail split-K plan of the SM-pair GATE_RES GEMM (host arithmetic only; pins the chooser in the CPU test-suite).
// out3 = {whole tiles, K segments per tail tile (1 = no split), K blocks of 64 per segment}
extern "C" int yb_gemm_splitk_plan(int tiles, int num_kb, int clusters, int split_k, int* out3) {
  if (tiles <= 0 || num_kb <= 0 || clusters <= 0 || split_k < 0 || split_k > 12 || !out3) return YB_ERR_ARG;
  yb::gemm_splitk_plan(tiles, num_kb, clusters, split_k, &out3[0], &out3[1], &out3[2]);
  return YB_OK;
}

// Bytes of caller-owned workspace yb_gemm_bf16 needs to split the tail of this launch (0 = it will not split). Asks the driver for
// the number of resident CTA pairs, so it needs a current device.
extern "C" long long yb_gemm_workspace_bytes(int M, int N, int K, int epilogue, int cta_pair, int split_k) {
  using namespace yb;
  if (M <= 0 || N <= 0 || K <= 0 || epilogue != YB_EPI_GATE_RES || split_k == 1 || split_k < 0 || split_k > 12) return 0;
  if (cta_pair != 2) return 0;   // only the SM-pair kernel splits
  static int max_clusters[kMaxDevices] = {0};
  static bool attr_set[kMaxDevices] = {false};
  const int dev = current_device();
  if (max_clusters[dev] == 0) {   // same query, same kernel attributes as the launch path: the two plans must agree
    if (ensure_dynamic_smem(gemm_kernel<YB_EPI_GATE_RES, 0, 2, 256>, GEMM_SMEM_BYTES, attr_set, "gemm")) return 0;
    max_clusters[dev] = pair_max_clusters(gemm_kernel<YB_EPI_GATE_RES, 0, 2, 256>);
  }
  const int bn = pair_block_n(M, N, max_clusters[dev]);
  const int tiles = ((M + 255) / 256) * ((N + bn - 1) / bn);
  int full, ns, per;
  gemm_splitk_plan(tiles, (K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K, max_clusters[dev], split_k, &full, &ns, &per);
  return static_cast<long long>(tiles - full) * ns * 256 * bn * 4;
}

extern "C" int yb_gemm_bf16(const yb_gemm_args* a, void* stream_) {
  using namespace yb;
  if (!a || !a->A || !a->B || !a->out) return YB_ERR_ARG;
  if (a->M <= 0 || a->N <= 0 || a->K <= 0) return YB_ERR_ARG;
  if (a->N % 32 != 0 || a->K % 8 != 0) return YB_ERR_SHAPE;
  if (a->epilogue < 0 || a->epilogue > YB_EPI_RES_BF16) return YB_ERR_ARG;
  if (a->epilogue == YB_EPI_RES_BF16 && (!a->res || (a->res_ld % 8))) return YB_ERR_ARG;
  if ((a->lda % 8) || (a->ldb % 8) || (a->ldo % 8) || (reinterpret_cast<uintptr_t>(a->out) & 0xF)) return YB_ERR_ALIGNMENT;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (a->struct_bytes != sizeof(yb_gemm_args)) return YB_ERR_ARG;   // caller compiled against another layout of the struct
  if (a->cta_pair < 0 || a->cta_pair > 2 || a->split_k < 0 || a->split_k > 12) return YB_ERR_ARG;
  int a_split = a->K;
  long long a_chunk_ld = 0;
  if (a->a_split > 0) {
    if (a->a_split % GEMM_BLOCK_K != 0 || a->K % a->a_split != 0) return YB_ERR_SHAPE;
    a_split = a->a_split;
    a_chunk_ld = a->a_split_stride;
  }
  const int a_chunks = a->K / a_split;
  if (a->n_split < 0 || (a->n_split > 0 && (a->n_split % 32 != 0 || a->epilogue != YB_EPI_BF16))) return YB_ERR_ARG;
  GemmParams p;
  p.M = a->M;
  p.N = a->N;
  p.K = a->K;
  p.bias = static_cast<const float*>(a->bias);
  p.out = a->out;
  p.ldo = a->ldo;
  p.gate = static_cast<const float*>(a->gate);
  p.gate_ld = a->gate_ld;
  p.tok_idx = static_cast<const int*>(a->tok_idx);
  p.a_split = a_split;
  p.res = static_cast<const __nv_bfloat16*>(a->res);
  p.res_ld = a->res_ld;
  p.conv = 0;
  p.n_split = a->n_split;
  p.split_stride = a->split_stride;
  p.block_n = 0;
  p.stages = 0;
  CUtensorMap tmA, tmB;
  int rc = make_tmap_bf16_3d(&tmA, a->A, a_chunks, a->M, a_split, a->lda, a_chunks > 1 ? a_chunk_ld : a->lda * (long long)a->M + 8,
                             GEMM_BLOCK_M, GEMM_BLOCK_K);
  if (rc) return rc;
  // SM-pair kernel only when asked for (see yb_gemm_plan)
  const bool pair = a->cta_pair == 2;
  if (pair) {
    int bn = a->block_n;
    if (bn == 0) bn = pair_block_n(a->M, a->N, sm_count() / 2);
    if (bn < 32 || bn > 256 || bn % 32 != 0) return YB_ERR_ARG;
    p.block_n = bn;
    rc = make_tmap_bf16_2d(&tmB, a->B, a->N, a->K, a->ldb, bn / 2, GEMM_BLOCK_K);
    if (rc) return rc;
    switch (a->epilogue) {
      case YB_EPI_BF16: return launch_gemm<YB_EPI_BF16, 0, 2>(tmA, tmB, nullptr, p, stream);
      case YB_EPI_GELU_BF16: return launch_gemm<YB_EPI_GELU_BF16, 0, 2>(tmA, tmB, nullptr, p, stream);
      case YB_EPI_F32: return launch_gemm<YB_EPI_F32, 0, 2>(tmA, tmB, nullptr, p, stream);
      case YB_EPI_GELU_ERF_BF16: return launch_gemm<YB_EPI_GELU_ERF_BF16, 0, 2>(tmA, tmB, nullptr, p, stream);
      case YB_EPI_RES_BF16: return launch_gemm<YB_EPI_RES_BF16, 0, 2>(tmA, tmB, nullptr, p, stream);
      default: return launch_gemm<YB_EPI_GATE_RES, 0, 2>(tmA, tmB, nullptr, p, stream, a->split_k, a->ws, a->ws_bytes);
    }
  }
  const int block_n = (a->block_n == 128 || a->block_n == 256) ? a->block_n : ((a->N % 256 == 0 || a->N > 1024) ? 256 : 128);
  rc = make_tmap_bf16_2d(&tmB, a->B, a->N, a->K, a->ldb, block_n, GEMM_BLOCK_K);
  if (rc) return rc;
  p.block_n = block_n;
  // TMA epilogue for a plain [M, N] output (the row pitch and base were checked above); the N-split layout and RES_BF16 keep the
  // register epilogue
  CUtensorMap tmO;
  const CUtensorMap* tmo = nullptr;
  if (a->n_split == 0 && a->epilogue != YB_EPI_RES_BF16) {
    const int elem = (a->epilogue == YB_EPI_F32 || a->epilogue == YB_EPI_GATE_RES) ? 4 : 2;
    rc = make_tmap_out_2d(&tmO, a->out, a->M, a->N, a->ldo, elem, 64);
    if (rc) return rc;
    tmo = &tmO;
  }
  switch (a->epilogue) {
    case YB_EPI_BF16: return launch_gemm<YB_EPI_BF16, 0, 1>(tmA, tmB, tmo, p, stream);
    case YB_EPI_GELU_BF16: return launch_gemm<YB_EPI_GELU_BF16, 0, 1>(tmA, tmB, tmo, p, stream);
    case YB_EPI_F32: return launch_gemm<YB_EPI_F32, 0, 1>(tmA, tmB, tmo, p, stream);
    case YB_EPI_GELU_ERF_BF16: return launch_gemm<YB_EPI_GELU_ERF_BF16, 0, 1>(tmA, tmB, tmo, p, stream);
    case YB_EPI_RES_BF16: return launch_gemm<YB_EPI_RES_BF16, 0, 1>(tmA, tmB, nullptr, p, stream);
    default: return launch_gemm<YB_EPI_GATE_RES, 0, 1>(tmA, tmB, tmo, p, stream);
  }
}


// Causal 3x3x3 conv (replicate padding) as an implicit GEMM on the same kernel. See include/yume_b200.h.
// t_hist > 0 is the history form (include/yume_b200_stream.h): the input holds t_hist carried frames in front of the T new ones,
// and those frames take the place of the causal zero padding in time (the tensor map spans all t_hist + T frames).
// rows is the row-halo form (include/yume_b200_vae_rows.h): the input has H + 2 rows, the two outer ones the neighbours' halo
// rows, and output row h reads input rows h .. h + 2 (no zero fill in H; the tile plan is the one of the H output rows).
// down is its strided form (include/yume_b200_vae_rows_enc.h): the map starts at row 1 of the band buffer and spans H + 1 rows,
// the last the halo row below, with the buffer's frame pitch; output row h reads map rows 2h .. 2h + 2 as the full-height map does.
enum ConvRows { kConvFull = 0, kConvRows = 1, kConvRowsDown = 2 };
static int conv3d_launch(const yb_conv3d_args* a, int t_hist, ConvRows form, void* stream_) {
  const bool rows = form == kConvRows, down = form == kConvRowsDown;
  using namespace yb;
  if (!a || !a->xpad || !a->w || !a->out) return YB_ERR_ARG;
  if (a->struct_bytes != sizeof(yb_conv3d_args)) return YB_ERR_ARG;
  if (a->T <= 0 || a->H <= 0 || a->W <= 0 || a->Cp <= 0 || a->Cout <= 0) return YB_ERR_ARG;
  if (t_hist < 0) return YB_ERR_ARG;
  if (a->Cp % 64 != 0 || a->Cout % 32 != 0) return YB_ERR_SHAPE;
  if ((a->ldo % 8) || (reinterpret_cast<uintptr_t>(a->out) & 0xF)) return YB_ERR_ALIGNMENT;
  if (a->epilogue != YB_EPI_BF16 && a->epilogue != YB_EPI_F32 && a->epilogue != YB_EPI_RES_BF16) return YB_ERR_ARG;
  if (a->epilogue == YB_EPI_RES_BF16 && (!a->res || (a->res_ld % 8))) return YB_ERR_ARG;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  GemmParams p;
  const int kt = a->kt > 0 ? a->kt : 3, kh = a->kh > 0 ? a->kh : 3, kw = a->kw > 0 ? a->kw : 3;
  if ((kt != 1 && kt != 3) || (kh != 1 && kh != 3) || (kw != 1 && kw != 3)) return YB_ERR_SHAPE;
  const int block_n = (a->Cout % 256 == 0) ? 256 : 128;
  bool fuse_w = false;
  if (a->cta_pair < 0 || a->cta_pair > 2) return YB_ERR_ARG;
  // strided form (the Encoder3d `Resample` convs): input extents T/H/W, output extents (in + pad - k) / stride + 1 with the
  // padding BEHIND the data (ZeroPad2d((0,1,0,1)), vae2_2.py:101-104) or none at all (time_conv, :105-110)
  const int st_t = a->stride_t > 0 ? a->stride_t : 1, st_hw = a->stride_hw > 0 ? a->stride_hw : 1;
  if (st_t > 2 || st_hw > 2) return YB_ERR_ARG;
  const bool strided = st_t > 1 || st_hw > 1;
  if (strided && !a->oob_zero_pad) return YB_ERR_ARG;
  // history: exactly the kt-1 frames of the causal pad (unit stride), or the one frame the stride-2 time_conv carries
  if (t_hist > 0 && (!a->oob_zero_pad || t_hist != (st_t > 1 ? 1 : kt - 1))) return YB_ERR_ARG;
  if (rows && (!a->oob_zero_pad || strided || kh != 3)) return YB_ERR_ARG;
  if (down && (!a->oob_zero_pad || st_hw != 2 || st_t != 1 || kt != 1 || kh != 3 || kw != 3 || t_hist || (a->H % 2)))
    return YB_ERR_ARG;
  const int inT = a->T + t_hist;   // frames the tensor map spans
  int oT = a->T, oH = a->H, oW = a->W;
  if (st_t > 1) oT = (inT - kt) / st_t + 1;
  if (st_hw > 1) { oH = (a->H + 1 - kh) / st_hw + 1; oW = (a->W + 1 - kw) / st_hw + 1; }
  if (oT <= 0 || oH <= 0 || oW <= 0) return YB_ERR_SHAPE;
  // SM-pair kernel: 1 = forced; 0 (automatic) and 2 run the 1-CTA kernel, the faster of the two on the H100 (see yb_gemm_plan)
  const bool conv_pair = a->cta_pair == 1;
  conv_plan(oT, oH, oW, block_n, kw, (conv_pair || strided) ? 1 : a->fuse_w, &p.TW, &p.TH, &p.TT, &fuse_w);
  p.tiles_w = (oW + p.TW - 1) / p.TW;
  p.tiles_h = (oH + p.TH - 1) / p.TH;
  const int tiles_t = (oT + p.TT - 1) / p.TT;
  const int taps = kt * kh * kw;
  p.conv = fuse_w ? 2 : 1;
  p.cin_chunks = a->Cp / 64;
  p.cT = oT; p.cH = oH; p.cW = oW;
  p.kh = kh; p.kw = kw;
  p.st_t = st_t; p.st_h = st_hw; p.st_w = st_hw;
  p.off_t = (a->oob_zero_pad && st_t == 1) ? kt - 1 - t_hist : 0;
  p.off_h = (a->oob_zero_pad && st_hw == 1 && !rows) ? kh / 2 : 0;
  p.off_w = (a->oob_zero_pad && st_hw == 1) ? kw / 2 : 0;
  p.out_t_mul = a->out_t_mul > 0 ? a->out_t_mul : 1;
  p.out_t_add = a->out_t_add;
  p.M = oT * oH * oW;
  p.N = a->Cout;
  p.K = taps * a->Cp;
  p.num_m_tiles = tiles_t * p.tiles_h * p.tiles_w;
  p.bias = static_cast<const float*>(a->bias);
  p.out = a->out;
  p.ldo = a->ldo;
  p.gate = nullptr; p.gate_ld = 0; p.tok_idx = nullptr;
  p.a_split = p.K; p.n_split = 0; p.split_stride = 0;
  p.res = static_cast<const __nv_bfloat16*>(a->res);
  p.res_ld = a->res_ld;
  CUtensorMap tmA, tmB;
  const int padT = a->oob_zero_pad ? 0 : kt - 1, padH = a->oob_zero_pad ? 0 : kh - 1, padW = a->oob_zero_pad ? 0 : kw - 1;
  const uint64_t row_elems = static_cast<uint64_t>(a->W) * a->Cp;
  int rc = down ? make_tmap_bf16_4d(&tmA, static_cast<const __nv_bfloat16*>(a->xpad) + row_elems, inT, a->H + 1, a->W, a->Cp,
                                    p.TT, p.TH, p.TW, 64, st_t, st_hw, st_hw, (a->H + 2) * row_elems)
                : make_tmap_bf16_4d(&tmA, a->xpad, inT + padT, a->H + (rows ? 2 : padH), a->W + padW, a->Cp, p.TT, p.TH,
                                    fuse_w ? CONVW_ROWS : p.TW, 64, st_t, st_hw, st_hw);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmB, a->w, a->Cout, static_cast<uint64_t>(taps) * a->Cp, static_cast<uint64_t>(taps) * a->Cp,
                         block_n, GEMM_BLOCK_K);
  if (rc) return rc;
  // SM-pair kernel (un-fused taps; each CTA of the pair owns one 128-voxel box, the weight tile is split between them)
  if (conv_pair && !fuse_w) {
    p.conv = 1;
    p.block_n = a->Cout <= 256 ? a->Cout : (a->Cout % 192 == 0 ? 192 : 256);
    CUtensorMap tmBp;
    rc = make_tmap_bf16_2d(&tmBp, a->w, a->Cout, static_cast<uint64_t>(taps) * a->Cp, static_cast<uint64_t>(taps) * a->Cp,
                           p.block_n / 2, GEMM_BLOCK_K);
    if (rc) return rc;
    switch (a->epilogue) {
      case YB_EPI_BF16: return launch_gemm<YB_EPI_BF16, 0, 2>(tmA, tmBp, nullptr, p, stream);
      case YB_EPI_F32: return launch_gemm<YB_EPI_F32, 0, 2>(tmA, tmBp, nullptr, p, stream);
      default: return launch_gemm<YB_EPI_RES_BF16, 0, 2>(tmA, tmBp, nullptr, p, stream);
    }
  }
  p.block_n = block_n;
#define YB_CONV_DISPATCH(CW)                                                                  \
  switch (a->epilogue) {                                                                     \
    case YB_EPI_BF16: return launch_gemm<YB_EPI_BF16, CW, 1>(tmA, tmB, nullptr, p, stream);   \
    case YB_EPI_F32: return launch_gemm<YB_EPI_F32, CW, 1>(tmA, tmB, nullptr, p, stream);     \
    default: return launch_gemm<YB_EPI_RES_BF16, CW, 1>(tmA, tmB, nullptr, p, stream);        \
  }
  if (fuse_w) {
    YB_CONV_DISPATCH(1)
  } else {
    YB_CONV_DISPATCH(0)
  }
#undef YB_CONV_DISPATCH
}

extern "C" int yb_conv3d_causal(const yb_conv3d_args* a, void* stream) { return conv3d_launch(a, 0, kConvFull, stream); }

extern "C" int yb_conv3d_causal_hist(const yb_conv3d_args* a, int t_hist, void* stream) {
  if (t_hist <= 0) return YB_ERR_ARG;
  return conv3d_launch(a, t_hist, kConvFull, stream);
}

extern "C" int yb_conv3d_rows(const yb_conv3d_args* a, int t_hist, void* stream) {
  return conv3d_launch(a, t_hist, kConvRows, stream);
}

extern "C" int yb_conv3d_rows_down(const yb_conv3d_args* a, void* stream) {
  return conv3d_launch(a, 0, kConvRowsDown, stream);
}
