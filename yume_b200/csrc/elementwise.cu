// elementwise.cu — the HBM-bound glue of the denoise path, each fused so the fp32 residual stream is read once
// per use: LayerNorm+adaLN modulate, RMSNorm+RoPE, patchify / unpatchify gathers, timestep embedding pieces
// and the small fp32 linears the reference keeps in fp32 (time MLP, head).
#include "yb_host.h"
#include "yb_ptx.cuh"

namespace yb {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum for blockDim.x == 256 (8 warps); `red` is 8 floats of smem. Result broadcast to all threads.
__device__ __forceinline__ float block_sum_256(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();  // protect `red` from the previous use
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (lane < 8) ? red[lane] : 0.f;
  t = warp_sum(t);
  return t;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm (+ optional affine) + adaLN modulate. One CTA (256 threads) per token row; the row lives in
// registers (C <= 8192 -> at most 8 float4 per thread), two-pass mean/variance in fp32 like
// nn.LayerNorm (reference: wan23/modules/model.py:140-150, 301, 310, 343-347).
// Algorithmic bytes per token: 4*C read + 2*C (bf16) or 4*C (f32) written.
// ------------------------------------------------------------------------------------------------
constexpr int LN_THREADS = 256;
constexpr int LN_MAX_VEC = 8;

template <bool OUT_F32>
__global__ void __launch_bounds__(LN_THREADS)
ln_modulate_kernel(const float* __restrict__ x, long long ldx, void* __restrict__ out, long long ldo,
                   const float* __restrict__ scale, const float* __restrict__ shift, long long mod_ld,
                   const int* __restrict__ tok_idx, const float* __restrict__ weight,
                   const float* __restrict__ lnbias, int C, float eps) {
  __shared__ float red[8];
  const int row = blockIdx.x;
  const int nvec = C >> 2;  // float4 per row
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<long long>(row) * ldx);
  float4 v[LN_MAX_VEC];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    const int idx = threadIdx.x + i * LN_THREADS;
    if (idx < nvec) {
      v[i] = xr[idx];
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  const float mean = block_sum_256(s, red) / static_cast<float>(C);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    const int idx = threadIdx.x + i * LN_THREADS;
    if (idx < nvec) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float var = block_sum_256(q, red) / static_cast<float>(C);
  const float rstd = rsqrtf(var + eps);
  const long long u = tok_idx ? tok_idx[row] : 0;
  const float4* sc4 = scale ? reinterpret_cast<const float4*>(scale + u * mod_ld) : nullptr;
  const float4* sh4 = shift ? reinterpret_cast<const float4*>(shift + u * mod_ld) : nullptr;
  const float4* w4 = weight ? reinterpret_cast<const float4*>(weight) : nullptr;
  const float4* b4 = lnbias ? reinterpret_cast<const float4*>(lnbias) : nullptr;
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    const int idx = threadIdx.x + i * LN_THREADS;
    if (idx < nvec) {
      float4 y;
      y.x = (v[i].x - mean) * rstd;
      y.y = (v[i].y - mean) * rstd;
      y.z = (v[i].z - mean) * rstd;
      y.w = (v[i].w - mean) * rstd;
      if (w4) {
        const float4 w = __ldg(w4 + idx);
        y.x *= w.x; y.y *= w.y; y.z *= w.z; y.w *= w.w;
      }
      if (b4) {
        const float4 b = __ldg(b4 + idx);
        y.x += b.x; y.y += b.y; y.z += b.z; y.w += b.w;
      }
      if (sc4) {
        const float4 c = __ldg(sc4 + idx);
        y.x *= (1.f + c.x); y.y *= (1.f + c.y); y.z *= (1.f + c.z); y.w *= (1.f + c.w);
      }
      if (sh4) {
        const float4 h = __ldg(sh4 + idx);
        y.x += h.x; y.y += h.y; y.z += h.z; y.w += h.w;
      }
      if (OUT_F32) {
        reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + static_cast<long long>(row) * ldo)[idx] = y;
      } else {
        uint2 w;
        w.x = pack_bf16x2(y.x, y.y);
        w.y = pack_bf16x2(y.z, y.w);
        reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + static_cast<long long>(row) * ldo)[idx] = w;
      }
    }
  }
}

// Read-only 16-byte load the compiler may NOT move (volatile + memory clobber). The norm/RoPE kernels below hold a whole
// token row in registers; left to itself the scheduler hoists the weight and angle loads of ALL chunks to the top of the
// apply loop (4 float4 per chunk: +192 registers at C = 3072 -> 255 registers and spills). With ordered loads the loop is a
// hand-made two-stage pipeline: the operands of chunk i+1 are in flight while chunk i is computed and stored.
__device__ __forceinline__ float4 ldg_f4_ordered(const float* p) {
  float4 v;
  asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}

// Warp-per-row variant for C = 128*NV (3072 -> NV 24, 5120 -> NV 40): the whole row lives in one warp's registers,
// reductions are shuffles only (no block barrier), and every lane keeps NV*16 bytes of loads in flight.
// One multiplicative and one additive per-column operand: (1 + scale[tok], shift[tok]) for adaLN (ADA = true) or the affine
// (weight, bias) of norm3 / MLPProj (ADA = false) — the host sends the rare "both" case to the general kernel.
template <int NV, bool OUT_F32, bool ADA>
__global__ void __launch_bounds__(256, (NV <= 24 && !OUT_F32 && ADA) ? 2 : 1)   // C <= 3072, bf16 out: <= 128 registers, two CTAs (16 rows) per SM
ln_modulate_warp_kernel(const float* __restrict__ x, long long ldx, void* __restrict__ out, long long ldo,
                        const float* __restrict__ mul, const float* __restrict__ add, long long mod_ld,
                        const int* __restrict__ tok_idx, int L, float eps) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= L) return;
  constexpr int C = NV * 128;
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<long long>(row) * ldx);
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = xr[lane + i * 32];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) * (1.0f / C);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.0f / C) + eps);
  const long long u = (ADA && tok_idx) ? tok_idx[row] : 0;
  // per-chunk operands through ORDERED loads: unordered, the scheduler hoists all 2 x NV of them above
  // the loop (198 registers at C = 3072 -> one CTA per SM)
  const float* mp = mul ? mul + u * mod_ld + lane * 4 : nullptr;
  const float* ap = add ? add + u * mod_ld + lane * 4 : nullptr;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int idx = lane + i * 32;
    float4 cm = make_float4(0.f, 0.f, 0.f, 0.f), ca = cm;
    if (mp) cm = ldg_f4_ordered(mp + i * 128);     // (L1 hits: every warp of the SM reads the same table rows; the other
    if (ap) ca = ldg_f4_ordered(ap + i * 128);     //  15 resident warps cover the latency)
    float4 y;
    y.x = (v[i].x - mean) * rstd;
    y.y = (v[i].y - mean) * rstd;
    y.z = (v[i].z - mean) * rstd;
    y.w = (v[i].w - mean) * rstd;
    if (mp) {
      if (ADA) { y.x *= (1.f + cm.x); y.y *= (1.f + cm.y); y.z *= (1.f + cm.z); y.w *= (1.f + cm.w); }
      else { y.x *= cm.x; y.y *= cm.y; y.z *= cm.z; y.w *= cm.w; }
    }
    if (ap) { y.x += ca.x; y.y += ca.y; y.z += ca.z; y.w += ca.w; }
    if (OUT_F32) {
      reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + static_cast<long long>(row) * ldo)[idx] = y;
    } else {
      uint2 w;
      w.x = pack_bf16x2(y.x, y.y);
      w.y = pack_bf16x2(y.z, y.w);
      reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + static_cast<long long>(row) * ldo)[idx] = w;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// WanRMSNorm over the full C row + weight + RoPE, in place on bf16 (reference: wan23/modules/model.py:121-137,
// 38-118). One CTA (256 threads) per token; thread handles 8-element (16 B) chunks, i.e. 4 RoPE pairs.
// rope table: float2 (cos, sin) [L, D/2]; pair j of each head = elements (2j, 2j+1)  (view_as_complex, :62-63).
// Algorithmic bytes per token: 2*C read + 2*C written (+ D*4 of table).
// ------------------------------------------------------------------------------------------------
constexpr int RR_THREADS = 256;
constexpr int RR_MAX_CHUNK = 4;  // C <= 8192

__global__ void __launch_bounds__(RR_THREADS)
rmsnorm_rope_kernel(__nv_bfloat16* __restrict__ qk, long long ld, int piece_cols, long long piece_stride,
                    const float* __restrict__ weight,
                    const float2* __restrict__ rope, int rope_len, int C, int D, float eps) {
  __shared__ float red[8];
  const int row = blockIdx.x;
  __nv_bfloat16* xrow = qk + static_cast<long long>(row) * ld;
  // chunk idx (8 elements at column idx*8) lives in piece (col / piece_cols) at offset col % piece_cols
  auto chunk_ptr = [&](int idx) -> uint4* {
    const int col = idx << 3;
    const int piece = col / piece_cols;
    return reinterpret_cast<uint4*>(xrow + piece * piece_stride + (col - piece * piece_cols));
  };
  const int nchunk = C >> 3;
  uint4 raw[RR_MAX_CHUNK];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < RR_MAX_CHUNK; ++i) {
    const int idx = threadIdx.x + i * RR_THREADS;
    if (idx < nchunk) {
      raw[i] = *chunk_ptr(idx);
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw[i]);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = __bfloat1622float2(h[k]);
        ss += f.x * f.x + f.y * f.y;
      }
    }
  }
  const float rstd = rsqrtf(block_sum_256(ss, red) / static_cast<float>(C) + eps);
  const bool rot = (rope != nullptr) && (row < rope_len);
  const int half = D >> 1;
#pragma unroll
  for (int i = 0; i < RR_MAX_CHUNK; ++i) {
    const int idx = threadIdx.x + i * RR_THREADS;
    if (idx < nchunk) {
      const int col = idx << 3;
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw[i]);
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(weight + col));
      const float4 w1 = __ldg(reinterpret_cast<const float4*>(weight + col + 4));
      const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
      const int pair0 = (col % D) >> 1;
      uint32_t o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = __bfloat1622float2(h[k]);
        float a = f.x * rstd * wv[2 * k];
        float b = f.y * rstd * wv[2 * k + 1];
        if (rot) {
          const float2 cs = __ldg(rope + static_cast<long long>(row) * half + pair0 + k);
          const float ra = a * cs.x - b * cs.y;
          const float rb = a * cs.y + b * cs.x;
          a = ra;
          b = rb;
        }
        o[k] = pack_bf16x2(a, b);
      }
      *chunk_ptr(idx) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

// Warp-per-row variant for C = 256*NCH (3072 -> 12, 5120 -> 20): NCH 16-byte chunks per lane.
template <int NCH>
__global__ void __launch_bounds__(256, (NCH <= 12) ? 2 : 1)   // C <= 3072: <= 128 registers, two CTAs per SM
rmsnorm_rope_warp_kernel(__nv_bfloat16* __restrict__ qk, long long ld, int piece_cols, long long piece_stride,
                         const float* __restrict__ weight, const float2* __restrict__ rope, int rope_len, int L, int D,
                         float eps) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= L) return;
  constexpr int C = NCH * 256;
  __nv_bfloat16* xrow = qk + static_cast<long long>(row) * ld;
  auto chunk_ptr = [&](int i) -> uint4* {
    const int col = (lane + i * 32) << 3;
    const int piece = col / piece_cols;
    return reinterpret_cast<uint4*>(xrow + piece * piece_stride + (col - piece * piece_cols));
  };
  uint4 raw[NCH];
#pragma unroll
  for (int i = 0; i < NCH; ++i) raw[i] = *chunk_ptr(i);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw[i]);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = __bfloat1622float2(h[k]);
      ss += f.x * f.x + f.y * f.y;
    }
  }
  const float rstd = rsqrtf(warp_sum(ss) * (1.0f / C) + eps);
  const bool rot = (rope != nullptr) && (row < rope_len);
  const int half = D >> 1;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int col = (lane + i * 32) << 3;
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw[i]);
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(weight + col));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(weight + col + 4));
    const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
    const int pair0 = (col % D) >> 1;
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = __bfloat1622float2(h[k]);
      float a = f.x * rstd * wv[2 * k];
      float b = f.y * rstd * wv[2 * k + 1];
      if (rot) {
        const float2 cs = __ldg(rope + static_cast<long long>(row) * half + pair0 + k);
        const float ra = a * cs.x - b * cs.y;
        const float rb = a * cs.y + b * cs.x;
        a = ra;
        b = rb;
      }
      o[k] = pack_bf16x2(a, b);
    }
    *chunk_ptr(i) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// q AND k of a token row in one launch (WanSelfAttention: norm_q(q), norm_k(k), then rope_apply on both with the SAME
// per-token angles — wan23/modules/model.py:190-200). One warp per token handles the q row, then the k row (the second
// pass finds the token's (cos, sin) row in L1); the (cos, sin) quads are fetched as float4 = two pairs. Replaces two
// rmsnorm_rope launches per block.
template <int NCH>
__global__ void __launch_bounds__(256, (NCH <= 12) ? 2 : 1)
qk_norm_rope_warp_kernel(__nv_bfloat16* __restrict__ q, __nv_bfloat16* __restrict__ k, long long ld,
                         const float* __restrict__ wq, const float* __restrict__ wk,
                         const float2* __restrict__ rope, int rope_len, int L, int D, float eps, int nparts) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= L) return;
  constexpr int C = NCH * 256;
  const long long row_off = static_cast<long long>(row) * ld + (lane << 3);
  auto chunk_off = [&](int i) -> long long { return row_off + i * 256; };   // (plain rows: immediate offsets from one base)
  const bool rot = (rope != nullptr) && (row < rope_len);
  const float* rope_row = reinterpret_cast<const float*>(rope) + static_cast<long long>(row) * D;   // D/2 pairs x 2 floats
#pragma unroll 1
  for (int part = 0; part < nparts; ++part) {   // nparts = 1: a single row set (cross-attention q, context k)
    __nv_bfloat16* base = part == 0 ? q : k;
    const float* weight = part == 0 ? wq : wk;
    uint4 raw[NCH];
#pragma unroll
    for (int i = 0; i < NCH; ++i) raw[i] = *reinterpret_cast<const uint4*>(base + chunk_off(i));
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw[i]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __bfloat1622float2(h[j]);
        ss += f.x * f.x + f.y * f.y;
      }
    }
    const float rstd = rsqrtf(warp_sum(ss) * (1.0f / C) + eps);
    // 256 % D == 0 (checked by the host): a lane's 8 columns sit at the same offset inside a head for every chunk
    // ((lane*8 + i*256) % D == lane*8 % D), so its 4 (cos, sin) pairs are loop invariants — two float4 loads per row.
    // Weight chunks go through ordered loads, prefetched one chunk ahead.
    float cs[8] = {1.f, 0.f, 1.f, 0.f, 1.f, 0.f, 1.f, 0.f};
    if (rot) {
      const float4 r0 = ldg_f4_ordered(rope_row + ((lane << 3) % D));
      const float4 r1 = ldg_f4_ordered(rope_row + ((lane << 3) % D) + 4);
      cs[0] = r0.x; cs[1] = r0.y; cs[2] = r0.z; cs[3] = r0.w; cs[4] = r1.x; cs[5] = r1.y; cs[6] = r1.z; cs[7] = r1.w;
    }
    float4 w0 = ldg_f4_ordered(weight + (lane << 3)), w1 = ldg_f4_ordered(weight + (lane << 3) + 4);
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      float4 nw0 = w0, nw1 = w1;
      if (i + 1 < NCH) {
        nw0 = ldg_f4_ordered(weight + (lane << 3) + (i + 1) * 256);
        nw1 = ldg_f4_ordered(weight + (lane << 3) + (i + 1) * 256 + 4);
      }
      const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw[i]);
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __bfloat1622float2(h[j]);
        const float a = f.x * rstd * wv[2 * j];
        const float b2 = f.y * rstd * wv[2 * j + 1];
        o[j] = pack_bf16x2(a * cs[2 * j] - b2 * cs[2 * j + 1], a * cs[2 * j + 1] + b2 * cs[2 * j]);
      }
      *reinterpret_cast<uint4*>(base + chunk_off(i)) = make_uint4(o[0], o[1], o[2], o[3]);
      w0 = nw0; w1 = nw1;
    }
  }
}

// Ulysses send side fused with the exchange: one warp per local token reads its q | k | v row (standard [L, 3C]
// layout), applies RMSNorm + weight + RoPE to q and k, and stores every 16-byte chunk DIRECTLY into the receive
// buffer of the rank that owns that head ([P(src), Lp, q|k|v of heads/P] on the peer, NVLink peer pointer).
// Replaces rmsnorm_rope + the q/k/v all-to-all (wan23/distributed/ulysses.py:32-34 does 3 NCCL all_to_alls).
struct PeerPtrs {
  __nv_bfloat16* p[8];
};
struct PeerPtrsF {
  float* p[8];
};
template <int NCH>
__global__ void __launch_bounds__(256)
sp_scatter_qkv_kernel(const __nv_bfloat16* __restrict__ qkv, long long ld, const float* __restrict__ wq,
                      const float* __restrict__ wk, const float2* __restrict__ rope, int rope_len, int L, int D,
                      float eps, const PeerPtrs peers, int rank, int Lp, int Wh) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= L) return;
  constexpr int C = NCH * 256;
  const int W3 = 3 * Wh;
  const bool rot = (rope != nullptr) && (row < rope_len);
  const int half = D >> 1;
  const long long dst_row = (static_cast<long long>(rank) * Lp + row) * W3;
#pragma unroll 1
  for (int part = 0; part < 3; ++part) {
    const __nv_bfloat16* src = qkv + static_cast<long long>(row) * ld + part * C;
    uint4 raw[NCH];
#pragma unroll
    for (int i = 0; i < NCH; ++i) raw[i] = *reinterpret_cast<const uint4*>(src + ((lane + i * 32) << 3));
    float rstd = 1.f;
    if (part < 2) {
      float ss = 0.f;
#pragma unroll
      for (int i = 0; i < NCH; ++i) {
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw[i]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = __bfloat1622float2(h[k]);
          ss += f.x * f.x + f.y * f.y;
        }
      }
      rstd = rsqrtf(warp_sum(ss) * (1.0f / C) + eps);
    }
    const float* weight = part == 0 ? wq : wk;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int col = (lane + i * 32) << 3;
      uint4 o = raw[i];
      if (part < 2) {
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw[i]);
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(weight + col));
        const float4 w1 = __ldg(reinterpret_cast<const float4*>(weight + col + 4));
        const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
        const int pair0 = (col % D) >> 1;
        uint32_t ov[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = __bfloat1622float2(h[k]);
          float a = f.x * rstd * wv[2 * k];
          float b = f.y * rstd * wv[2 * k + 1];
          if (rot) {
            const float2 cs = __ldg(rope + static_cast<long long>(row) * half + pair0 + k);
            const float ra = a * cs.x - b * cs.y;
            const float rb = a * cs.y + b * cs.x;
            a = ra;
            b = rb;
          }
          ov[k] = pack_bf16x2(a, b);
        }
        o = make_uint4(ov[0], ov[1], ov[2], ov[3]);
      }
      const int peer = col / Wh;
      *reinterpret_cast<uint4*>(peers.p[peer] + dst_row + part * Wh + (col - peer * Wh)) = o;
    }
  }
}

// Receiver side of the fused projection + all-to-all (yb_gemm_sp_qkv): the q | k columns this rank received are still
// un-normalised (WanRMSNorm needs the sum of squares over ALL heads of a token, which no single rank holds).
//   sp_bcast_sums_kernel   every rank copies its [Lp][2] sums of squares (q, k) into slot `rank` of every peer's table and
//                          clears its accumulator for the next layer
//   sp_post_norm_rope_kernel  after the barrier: q, k <- bf16(rope(x * rstd(token) * weight[my heads])) in place on the
//                          received [L, 3*Wh] rows (one warp per token; v untouched) — the arithmetic of rmsnorm_rope, moved
//                          behind the exchange so that the NVLink traffic rides under the GEMM instead of a separate pass.
__global__ void sp_bcast_sums_kernel(float* __restrict__ local, const PeerPtrsF peers, int rank, int Lp) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Lp) return;
  const float2 v = reinterpret_cast<const float2*>(local)[i];
#pragma unroll
  for (int p = 0; p < 8; ++p)
    if (peers.p[p]) reinterpret_cast<float2*>(peers.p[p])[static_cast<long long>(rank) * Lp + i] = v;
  reinterpret_cast<float2*>(local)[i] = make_float2(0.f, 0.f);
}

__global__ void __launch_bounds__(256)
sp_post_norm_rope_kernel(__nv_bfloat16* __restrict__ buf, const float* __restrict__ sums, const float* __restrict__ wq,
                         const float* __restrict__ wk, const float2* __restrict__ rope, int rope_len, int L, int Wh, int C,
                         int D, float eps) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= L) return;
  const float2 ss = reinterpret_cast<const float2*>(sums)[row];
  const float rstd_q = rsqrtf(ss.x / static_cast<float>(C) + eps), rstd_k = rsqrtf(ss.y / static_cast<float>(C) + eps);
  const bool rot = (rope != nullptr) && (row < rope_len);
  const float* rope_row = reinterpret_cast<const float*>(rope) + static_cast<long long>(row) * D;
  __nv_bfloat16* base = buf + static_cast<long long>(row) * (3 * Wh);
  const int nch = Wh >> 3;
  for (int c = lane; c < 2 * nch; c += 32) {       // chunks [0, nch) = q, [nch, 2 nch) = k
    const int part = c >= nch ? 1 : 0;
    const int col = (c - part * nch) << 3;
    const float* weight = part ? wk : wq;
    const float rstd = part ? rstd_k : rstd_q;
    uint4 raw = *reinterpret_cast<const uint4*>(base + part * Wh + col);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(weight + col));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(weight + col + 4));
    const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
    float cs[8] = {1.f, 0.f, 1.f, 0.f, 1.f, 0.f, 1.f, 0.f};
    if (rot) {
      const float4 r0 = __ldg(reinterpret_cast<const float4*>(rope_row + (col % D)));
      const float4 r1 = __ldg(reinterpret_cast<const float4*>(rope_row + (col % D) + 4));
      cs[0] = r0.x; cs[1] = r0.y; cs[2] = r0.z; cs[3] = r0.w; cs[4] = r1.x; cs[5] = r1.y; cs[6] = r1.z; cs[7] = r1.w;
    }
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __bfloat1622float2(h[j]);
      const float a = f.x * rstd * wv[2 * j];
      const float b2 = f.y * rstd * wv[2 * j + 1];
      o[j] = pack_bf16x2(a * cs[2 * j] - b2 * cs[2 * j + 1], a * cs[2 * j + 1] + b2 * cs[2 * j]);
    }
    *reinterpret_cast<uint4*>(base + part * Wh + col) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// ------------------------------------------------------------------------------------------------
// patchify gather: x f32 [Cin, F, H, W] -> bf16 [L, Cin*ph*pw], token order (f, hp, wp), column order
// (cin, i, j) = Conv3d weight.flatten(1) order for kernel (1, ph, pw). Out-of-range H/W read as zero (convpadd).
// ------------------------------------------------------------------------------------------------
__global__ void patchify_kernel(const float* __restrict__ x, long long sc, long long sf, long long sh, long long sw,
                                __nv_bfloat16* __restrict__ out, long long ldo, int Cin, int F, int H, int W, int ph,
                                int pw, int Hp, int Wp) {
  const int Kc = Cin * ph * pw;
  const long long total = static_cast<long long>(F) * Hp * Wp * Kc;
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int kc = static_cast<int>(t % Kc);
    const long long tok = t / Kc;
    const int wp = static_cast<int>(tok % Wp);
    const int hp = static_cast<int>((tok / Wp) % Hp);
    const int f = static_cast<int>(tok / (static_cast<long long>(Wp) * Hp));
    const int j = kc % pw;
    const int i = (kc / pw) % ph;
    const int c = kc / (pw * ph);
    const int h = hp * ph + i, w = wp * pw + j;
    float v = 0.f;
    if (h < H && w < W) v = x[c * sc + f * sf + h * sh + w * sw];
    out[tok * ldo + kc] = __float2bfloat16_rn(v);
  }
}

// unpatchify: y f32 [L, ph*pw*Cout] -> out f32 [Cout, F, Hp*ph, Wp*pw]  ('fhwpqrc->cfphqwr', p == 1)
__global__ void unpatchify_kernel(const float* __restrict__ y, long long ldy, float* __restrict__ out, int Cout, int F,
                                  int Hp, int Wp, int ph, int pw) {
  const int Ho = Hp * ph, Wo = Wp * pw;
  const long long total = static_cast<long long>(Cout) * F * Ho * Wo;
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int w = static_cast<int>(t % Wo);
    const int h = static_cast<int>((t / Wo) % Ho);
    const int f = static_cast<int>((t / (static_cast<long long>(Wo) * Ho)) % F);
    const int c = static_cast<int>(t / (static_cast<long long>(Wo) * Ho * F));
    const int hp = h / ph, q = h % ph, wp = w / pw, r = w % pw;
    const long long tok = (static_cast<long long>(f) * Hp + hp) * Wp + wp;
    out[t] = y[tok * ldy + (static_cast<long long>(q) * pw + r) * Cout + c];
  }
}

// sinusoidal embedding in fp64 (reference: wan23/modules/model.py:14-24): out[n, :half] = cos, [half:] = sin
__global__ void sinusoidal_kernel(const float* __restrict__ t, float* __restrict__ out, int n, int dim) {
  const int half = dim >> 1;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * half) return;
  const int r = idx / half, i = idx % half;
  const double pos = static_cast<double>(t[r]);
  const double freq = pow(10000.0, -static_cast<double>(i) / static_cast<double>(half));
  const double a = pos * freq;
  out[static_cast<long long>(r) * dim + i] = static_cast<float>(cos(a));
  out[static_cast<long long>(r) * dim + half + i] = static_cast<float>(sin(a));
}

// small-M fp32 linear: one warp per output column n, all M (<= 16) rows at once. Weight-read bound.
constexpr int LS_MAX_M = 16;
__global__ void __launch_bounds__(256)
linear_f32_small_kernel(const float* __restrict__ in, const float* __restrict__ W, const float* __restrict__ bias,
                        float* __restrict__ out, int M, int N, int K, int silu_in) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  float acc[LS_MAX_M];
#pragma unroll
  for (int m = 0; m < LS_MAX_M; ++m) acc[m] = 0.f;
  const float* wr = W + static_cast<long long>(n) * K;
  for (int k = lane; k < K; k += 32) {
    const float w = __ldg(wr + k);
#pragma unroll
    for (int m = 0; m < LS_MAX_M; ++m) {
      if (m < M) {
        float a = in[static_cast<long long>(m) * K + k];
        if (silu_in) a = a / (1.f + expf(-a));
        acc[m] = fmaf(a, w, acc[m]);
      }
    }
  }
#pragma unroll
  for (int m = 0; m < LS_MAX_M; ++m) {
    if (m < M) {
      const float s = warp_sum(acc[m]);
      if (lane == 0) out[static_cast<long long>(m) * N + n] = s + (bias ? bias[n] : 0.f);
    }
  }
}

// general fp32 linear (SIMT): 64x64 output tile per CTA of 256 threads, 4x4 per thread, K step 16.
__global__ void __launch_bounds__(256)
linear_f32_kernel(const float* __restrict__ in, long long ldi, const float* __restrict__ W,
                  const float* __restrict__ bias, float* __restrict__ out, long long ldo, int M, int N, int K) {
  __shared__ float sa[16][64 + 4];
  __shared__ float sb[16][64 + 4];
  const int tm = blockIdx.y * 64, tn = blockIdx.x * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4] = {};
  const int lr = threadIdx.x >> 2;        // 0..63: row within the tile
  const int lk = (threadIdx.x & 3) << 2;  // 0,4,8,12: k offset
  for (int k0 = 0; k0 < K; k0 += 16) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (tm + lr < M && k0 + lk < K) a = *reinterpret_cast<const float4*>(in + static_cast<long long>(tm + lr) * ldi + k0 + lk);
    if (tn + lr < N && k0 + lk < K) b = __ldg(reinterpret_cast<const float4*>(W + static_cast<long long>(tn + lr) * K + k0 + lk));
    __syncthreads();
    sa[lk + 0][lr] = a.x; sa[lk + 1][lr] = a.y; sa[lk + 2][lr] = a.z; sa[lk + 3][lr] = a.w;
    sb[lk + 0][lr] = b.x; sb[lk + 1][lr] = b.y; sb[lk + 2][lr] = b.z; sb[lk + 3][lr] = b.w;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&sa[k][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&sb[k][tx * 4]);
      const float ar[4] = {av.x, av.y, av.z, av.w};
      const float br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = tm + ty * 4 + i;
    if (r >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = tn + tx * 4 + j;
      if (c < N) out[static_cast<long long>(r) * ldo + c] = acc[i][j] + (bias ? bias[c] : 0.f);
    }
  }
}

// out[r1][r2][:] = a[r1][:] + b[r2][:]  (per-block modulation tables: modulation[i] + e0[u], model.py:296)
__global__ void bcast_add_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out,
                                 int R1, int R2, int n) {
  const long long total = static_cast<long long>(R1) * R2 * n;
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(t % n);
    const int r2 = static_cast<int>((t / n) % R2);
    const int r1 = static_cast<int>(t / (static_cast<long long>(n) * R2));
    out[t] = a[static_cast<long long>(r1) * n + c] + b[static_cast<long long>(r2) * n + c];
  }
}

}  // namespace yb

using namespace yb;

extern "C" int yb_bcast_add(const void* a, const void* b, void* out, int R1, int R2, int n, void* stream_) {
  if (!a || !b || !out || R1 <= 0 || R2 <= 0 || n <= 0) return YB_ERR_ARG;
  const long long total = static_cast<long long>(R1) * R2 * n;
  const int blocks = static_cast<int>(total / 256 + 1 < static_cast<long long>(sm_count()) * 8 ? total / 256 + 1 : static_cast<long long>(sm_count()) * 8);
  bcast_add_kernel<<<blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(a), static_cast<const float*>(b), static_cast<float*>(out), R1, R2, n);
  return check_launch("bcast_add");
}

extern "C" int yb_abi_version(void) { return 4; }

extern "C" int yb_ln_modulate(const void* x, long long ldx, void* out, long long ldo, int out_f32, const void* scale,
                              const void* shift, long long mod_ld, const void* tok_idx, const void* weight,
                              const void* lnbias, int L, int C, float eps, void* stream_) {
  if (!x || !out || L <= 0 || C <= 0) return YB_ERR_ARG;
  if (C % 8 != 0 || C > LN_THREADS * LN_MAX_VEC * 4) return YB_ERR_SHAPE;
  if ((ldx % 4) || (ldo % 8) || (mod_ld % 4)) return YB_ERR_ALIGNMENT;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  const bool ada = scale || shift, affine = weight || lnbias;
#define YB_LN_LAUNCH(NV, F32, ADA, MUL, ADD)                                                                            \
  ln_modulate_warp_kernel<NV, F32, ADA><<<(L + 7) / 8, 256, 0, s>>>(static_cast<const float*>(x), ldx, out, ldo,         \
                                                                    static_cast<const float*>(MUL),                      \
                                                                    static_cast<const float*>(ADD), mod_ld,              \
                                                                    static_cast<const int*>(tok_idx), L, eps)
#define YB_LN_WARP(NV)                                                                                                  \
  if (C == (NV) * 128 && !(ada && affine)) {                                                                            \
    if (affine) {                                                                                                       \
      if (out_f32) YB_LN_LAUNCH(NV, true, false, weight, lnbias); else YB_LN_LAUNCH(NV, false, false, weight, lnbias);  \
    } else {                                                                                                            \
      if (out_f32) YB_LN_LAUNCH(NV, true, true, scale, shift); else YB_LN_LAUNCH(NV, false, true, scale, shift);        \
    }                                                                                                                   \
    return check_launch("ln_modulate");                                                                                 \
  }
  YB_LN_WARP(24)
  YB_LN_WARP(40)
  YB_LN_WARP(8)
  YB_LN_WARP(2)
#undef YB_LN_LAUNCH
#undef YB_LN_WARP
  if (out_f32)
    ln_modulate_kernel<true><<<L, LN_THREADS, 0, s>>>(static_cast<const float*>(x), ldx, out, ldo,
                                                      static_cast<const float*>(scale), static_cast<const float*>(shift),
                                                      mod_ld, static_cast<const int*>(tok_idx),
                                                      static_cast<const float*>(weight), static_cast<const float*>(lnbias),
                                                      C, eps);
  else
    ln_modulate_kernel<false><<<L, LN_THREADS, 0, s>>>(static_cast<const float*>(x), ldx, out, ldo,
                                                       static_cast<const float*>(scale), static_cast<const float*>(shift),
                                                       mod_ld, static_cast<const int*>(tok_idx),
                                                       static_cast<const float*>(weight), static_cast<const float*>(lnbias),
                                                       C, eps);
  return check_launch("ln_modulate");
}

extern "C" int yb_rmsnorm_rope_pieces(void* qk, long long ld, int piece_cols, long long piece_stride,
                                      const void* weight, const void* rope, int rope_len, int L, int C, int D,
                                      float eps, void* stream_) {
  if (!qk || !weight || L <= 0 || C <= 0 || D <= 0 || piece_cols <= 0) return YB_ERR_ARG;
  if (C % 8 != 0 || C > RR_THREADS * RR_MAX_CHUNK * 8 || D % 8 != 0 || C % D != 0) return YB_ERR_SHAPE;
  if (piece_cols % 8 != 0 || C % piece_cols != 0) return YB_ERR_SHAPE;
  if ((ld % 8) || (piece_stride % 8) || (reinterpret_cast<uintptr_t>(qk) & 0xF)) return YB_ERR_ALIGNMENT;
  // plain rows whose head_dim divides 256: the faster pass of yb_qk_norm_rope with one row set (ordered weight loads, the
  // (cos, sin) quad of a lane loaded once per row) — the cross-attention q rows and the context k rows
#define YB_RR_FAST(NCH)                                                                                              \
  if (C == (NCH) * 256 && piece_cols == C && 256 % D == 0) {                                                         \
    qk_norm_rope_warp_kernel<NCH><<<(L + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(                  \
        static_cast<__nv_bfloat16*>(qk), static_cast<__nv_bfloat16*>(qk), ld, static_cast<const float*>(weight),     \
        static_cast<const float*>(weight), static_cast<const float2*>(rope), rope_len, L, D, eps, 1);                \
    return check_launch("rmsnorm_rope");                                                                             \
  }
  YB_RR_FAST(12)
  YB_RR_FAST(20)
  YB_RR_FAST(4)
  YB_RR_FAST(1)
#undef YB_RR_FAST
#define YB_RR_WARP(NCH)                                                                                              \
  if (C == (NCH) * 256) {                                                                                            \
    rmsnorm_rope_warp_kernel<NCH><<<(L + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(                  \
        static_cast<__nv_bfloat16*>(qk), ld, piece_cols, piece_stride, static_cast<const float*>(weight),             \
        static_cast<const float2*>(rope), rope_len, L, D, eps);                                                       \
    return check_launch("rmsnorm_rope");                                                                             \
  }
  YB_RR_WARP(12)
  YB_RR_WARP(20)
  YB_RR_WARP(4)
  YB_RR_WARP(1)
#undef YB_RR_WARP
  rmsnorm_rope_kernel<<<L, RR_THREADS, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<__nv_bfloat16*>(qk), ld, piece_cols, piece_stride, static_cast<const float*>(weight),
      static_cast<const float2*>(rope), rope_len, C, D, eps);
  return check_launch("rmsnorm_rope");
}

extern "C" int yb_rmsnorm_rope(void* qk, long long ld, const void* weight, const void* rope, int rope_len, int L,
                               int C, int D, float eps, void* stream_) {
  return yb_rmsnorm_rope_pieces(qk, ld, C, 0, weight, rope, rope_len, L, C, D, eps, stream_);
}

// RMSNorm(q) | RMSNorm(k) + RoPE on both, one launch (see qk_norm_rope_warp_kernel). q / k: first element of the two
// [L, C] row sets (same row stride `ld`, same piece layout). Widths without a warp-per-row instance run the general
// kernel twice.
extern "C" int yb_qk_norm_rope(void* q, void* k, long long ld, int piece_cols, long long piece_stride, const void* wq,
                               const void* wk, const void* rope, int rope_len, int L, int C, int D, float eps,
                               void* stream_) {
  if (!q || !k || !wq || !wk || L <= 0 || C <= 0 || D <= 0 || piece_cols <= 0) return YB_ERR_ARG;
  if (C % 8 != 0 || D % 8 != 0 || C % D != 0 || piece_cols % 8 != 0 || C % piece_cols != 0) return YB_ERR_SHAPE;
  if ((ld % 8) || (piece_stride % 8) || (reinterpret_cast<uintptr_t>(q) & 0xF) || (reinterpret_cast<uintptr_t>(k) & 0xF))
    return YB_ERR_ALIGNMENT;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
#define YB_QK_WARP(NCH)                                                                                               \
  if (C == (NCH) * 256 && piece_cols == C && 256 % D == 0) {                                                                                             \
    qk_norm_rope_warp_kernel<NCH><<<(L + 7) / 8, 256, 0, s>>>(                                                         \
        static_cast<__nv_bfloat16*>(q), static_cast<__nv_bfloat16*>(k), ld,                                            \
        static_cast<const float*>(wq), static_cast<const float*>(wk), static_cast<const float2*>(rope), rope_len, L, D, \
        eps, 2);                                                                                                       \
    return check_launch("qk_norm_rope");                                                                              \
  }
  YB_QK_WARP(12)
  YB_QK_WARP(20)
  YB_QK_WARP(4)
  YB_QK_WARP(1)
#undef YB_QK_WARP
  int rc = yb_rmsnorm_rope_pieces(q, ld, piece_cols, piece_stride, wq, rope, rope_len, L, C, D, eps, stream_);
  if (rc) return rc;
  return yb_rmsnorm_rope_pieces(k, ld, piece_cols, piece_stride, wk, rope, rope_len, L, C, D, eps, stream_);
}

extern "C" int yb_patchify(const void* x, long long sc, long long sf, long long sh, long long sw, void* out,
                           long long ldo, int Cin, int F, int H, int W, int ph, int pw, void* stream_) {
  if (!x || !out || Cin <= 0 || F <= 0 || H <= 0 || W <= 0 || ph <= 0 || pw <= 0) return YB_ERR_ARG;
  const int Hp = (H + ph - 1) / ph, Wp = (W + pw - 1) / pw;
  const long long total = static_cast<long long>(F) * Hp * Wp * Cin * ph * pw;
  const int blocks = static_cast<int>(total / 256 + 1 < static_cast<long long>(sm_count()) * 16 ? total / 256 + 1 : static_cast<long long>(sm_count()) * 16);
  patchify_kernel<<<blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(x), sc, sf, sh, sw, static_cast<__nv_bfloat16*>(out), ldo, Cin, F, H, W, ph, pw, Hp,
      Wp);
  return check_launch("patchify");
}

extern "C" int yb_unpatchify(const void* y, long long ldy, void* out, int Cout, int F, int Hp, int Wp, int ph, int pw,
                             void* stream_) {
  if (!y || !out || Cout <= 0 || F <= 0 || Hp <= 0 || Wp <= 0 || ph <= 0 || pw <= 0) return YB_ERR_ARG;
  const long long total = static_cast<long long>(Cout) * F * Hp * ph * Wp * pw;
  const int blocks = static_cast<int>(total / 256 + 1 < static_cast<long long>(sm_count()) * 16 ? total / 256 + 1 : static_cast<long long>(sm_count()) * 16);
  unpatchify_kernel<<<blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(y), ldy, static_cast<float*>(out), Cout, F, Hp, Wp, ph, pw);
  return check_launch("unpatchify");
}

extern "C" int yb_sinusoidal(const void* t, void* out, int n, int dim, void* stream_) {
  if (!t || !out || n <= 0 || dim <= 0 || (dim & 1)) return YB_ERR_ARG;
  const int total = n * (dim / 2);
  sinusoidal_kernel<<<(total + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(t), static_cast<float*>(out), n, dim);
  return check_launch("sinusoidal");
}

extern "C" int yb_linear_f32_small(const void* in, const void* W, const void* bias, void* out, int M, int N, int K,
                                   int silu_in, void* stream_) {
  if (!in || !W || !out || M <= 0 || N <= 0 || K <= 0) return YB_ERR_ARG;
  if (M > LS_MAX_M) return YB_ERR_SHAPE;
  linear_f32_small_kernel<<<(N + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(in), static_cast<const float*>(W), static_cast<const float*>(bias),
      static_cast<float*>(out), M, N, K, silu_in);
  return check_launch("linear_f32_small");
}

extern "C" int yb_linear_f32(const void* in, long long ldi, const void* W, const void* bias, void* out, long long ldo,
                             int M, int N, int K, void* stream_) {
  if (!in || !W || !out || M <= 0 || N <= 0 || K <= 0) return YB_ERR_ARG;
  if ((K % 4) || (ldi % 4)) return YB_ERR_SHAPE;
  dim3 grid((N + 63) / 64, (M + 63) / 64);
  linear_f32_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(in), ldi, static_cast<const float*>(W), static_cast<const float*>(bias),
      static_cast<float*>(out), ldo, M, N, K);
  return check_launch("linear_f32");
}


extern "C" int yb_sp_bcast_sums(void* local, void* const* peers, int world, int rank, int Lp, void* stream_) {
  if (!local || !peers || world < 2 || world > 8 || rank < 0 || rank >= world || Lp <= 0) return YB_ERR_ARG;
  PeerPtrsF pp;
  for (int i = 0; i < 8; ++i) pp.p[i] = i < world ? static_cast<float*>(peers[i]) : nullptr;
  sp_bcast_sums_kernel<<<(Lp + 255) / 256, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(static_cast<float*>(local), pp, rank, Lp);
  return check_launch("sp_bcast_sums");
}

extern "C" int yb_sp_post_norm_rope(void* buf, const void* sums, const void* wq, const void* wk, const void* rope, int rope_len,
                                    int L, int Wh, int C, int D, float eps, void* stream_) {
  if (!buf || !sums || !wq || !wk || L <= 0 || Wh <= 0 || C <= 0 || D <= 0) return YB_ERR_ARG;
  if (Wh % D != 0 || D % 8 != 0 || (reinterpret_cast<uintptr_t>(buf) & 0xF)) return YB_ERR_SHAPE;
  sp_post_norm_rope_kernel<<<(L + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<__nv_bfloat16*>(buf), static_cast<const float*>(sums), static_cast<const float*>(wq),
      static_cast<const float*>(wk), static_cast<const float2*>(rope), rope_len, L, Wh, C, D, eps);
  return check_launch("sp_post_norm_rope");
}

extern "C" int yb_sp_scatter_qkv(const void* qkv, long long ld, const void* wq, const void* wk, const void* rope,
                                 int rope_len, int L, int C, int D, float eps, void* const* peers, int world, int rank,
                                 int Lp, void* stream_) {
  if (!qkv || !wq || !wk || !peers || L <= 0 || world < 2 || world > 8 || rank < 0 || rank >= world) return YB_ERR_ARG;
  if (C % (world * D) != 0 || (ld % 8)) return YB_ERR_SHAPE;
  PeerPtrs pp;
  for (int i = 0; i < 8; ++i) pp.p[i] = i < world ? static_cast<__nv_bfloat16*>(peers[i]) : nullptr;
  const int Wh = C / world;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
#define YB_SC(NCH)                                                                                                   \
  if (C == (NCH) * 256) {                                                                                            \
    sp_scatter_qkv_kernel<NCH><<<(L + 7) / 8, 256, 0, s>>>(static_cast<const __nv_bfloat16*>(qkv), ld,                \
                                                          static_cast<const float*>(wq), static_cast<const float*>(wk), \
                                                          static_cast<const float2*>(rope), rope_len, L, D, eps, pp,   \
                                                          rank, Lp, Wh);                                              \
    return check_launch("sp_scatter_qkv");                                                                           \
  }
  YB_SC(12)
  YB_SC(20)
  YB_SC(4)
  YB_SC(1)
#undef YB_SC
  return YB_ERR_SHAPE;
}
