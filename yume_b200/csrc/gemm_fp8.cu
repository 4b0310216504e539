// gemm_fp8.cu — the FP8 (e4m3) path of the DiT block GEMMs on sm_90a (H100): a block-scaled wgmma GEMM with per-group
// promotion, and the two kernels that produce its 1x128-quantised activations (LayerNorm + modulate, and bf16 rows).
// Numerics and constraints: include/yume_b200_fp8.h. Structure follows gemm.cu (persistent, warp-specialised, TMA ring):
//   warp 0 (one thread)  TMA producer: A tile 128 x 128 e4m3, B tile 128 x 128 e4m3 (128B swizzle: one 128-byte swizzle row is
//                        exactly one scale group) and the 128 A-scales of that k-group (512 B) into stage s of the ring
//   warpgroups 1-2       consumers, rows [64 * (wg - 1), +64): per k-group 4 x wgmma m64n128k32 into a fresh accumulator, wait,
//                        then promotion acc_p += s_a[row] * acc (fp32 FMA); epilogue straight from the fragment registers
#include "yb_host.h"
#include "../../include/yume_b200_fp8.h"
#include "yb_ptx.cuh"

namespace yb {

constexpr int F8_BLOCK_M = 128;
constexpr int F8_BLOCK_N = 128;
constexpr int F8_BLOCK_K = 128;                              // 128 e4m3 = 128 B = one swizzle row = one scale group
constexpr int F8_THREADS = 384;
constexpr int F8_GROUP_N = 8;                                // rasterisation as gemm.cu
constexpr int F8_TILE_BYTES = 128 * 128;                     // one operand tile
constexpr int F8_STAGES = 6;
constexpr int F8_SCALE_BYTES = F8_BLOCK_M * 4;
constexpr int F8_SMEM_BYTES = 1024 + F8_STAGES * (2 * F8_TILE_BYTES + F8_SCALE_BYTES) + 256;

__device__ __forceinline__ void f8_tile_coords(int tile, int num_m_tiles, int num_n_tiles, int& m_tile, int& n_tile) {
  const int per_group = F8_GROUP_N * num_m_tiles;
  const int g = tile / per_group;
  const int r = tile - g * per_group;
  const int n_first = g * F8_GROUP_N;
  const int n_in_group = min(F8_GROUP_N, num_n_tiles - n_first);
  m_tile = r / n_in_group;
  n_tile = n_first + (r - m_tile * n_in_group);
}

// D (64 x 128, fp32) (+)= A (64 x 32 e4m3, smem K-major) * B (128 x 32 e4m3, smem K-major); fragment layout as wgmma_ss_n128
__device__ __forceinline__ void wgmma_e4m3_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// two floats -> two e4m3 bytes (lo = first), round to nearest even, saturating to +-448, NaN kept
__device__ __forceinline__ uint16_t cvt_e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}

// (inv, scale) of a group with max |x| == amax (NaN excluded): see include/yume_b200_fp8.h
__device__ __forceinline__ void group_scale(float amax, float& inv, float& scale) {
  inv = __fdiv_rn(448.0f, amax);
  scale = __fdiv_rn(amax, 448.0f);
  if (!(inv <= 3.402823466e38f)) { inv = 0.f; scale = 0.f; }
}

// |x| for the group maximum: a NaN element does not take part (fmaxf returns the other operand)
__device__ __forceinline__ float amax4(float a, float b, float c, float d) {
  return fmaxf(fmaxf(fabsf(a), fabsf(b)), fmaxf(fabsf(c), fabsf(d)));
}

__device__ __forceinline__ float f8_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

struct Fp8Params {
  int M, N, K, num_m_tiles, num_n_tiles;
  const float* b_scale;
  const float* bias;
  void* out;
  long long ldo;
  float* out_scale;
  long long ldos;
  const float* gate;
  long long gate_ld;
  const int* tok_idx;
};

template <int EPI>
__global__ void __launch_bounds__(F8_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmS, const Fp8Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* sscale = reinterpret_cast<float*>(smem + F8_STAGES * 2 * F8_TILE_BYTES);   // [stage][128]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sscale + F8_STAGES * F8_BLOCK_M);
  uint64_t* empty_bar = full_bar + F8_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.num_m_tiles * p.num_n_tiles;
  const int num_kb = p.K / F8_BLOCK_K;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmS);
    for (int i = 0; i < F8_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);   // the 8 consumer warps
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      // ------------------------------- TMA producer -------------------------------
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_tile, n_tile;
        f8_tile_coords(tile, p.num_m_tiles, p.num_n_tiles, m_tile, n_tile);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * 2 * F8_TILE_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], 2 * F8_TILE_BYTES + F8_SCALE_BYTES);
          tma_load_2d(sa, &tmA, &full_bar[stage], kb * F8_BLOCK_K, m_tile * F8_BLOCK_M);
          tma_load_2d(sa + F8_TILE_BYTES, &tmB, &full_bar[stage], kb * F8_BLOCK_K, n_tile * F8_BLOCK_N);
          tma_load_2d(sscale + stage * F8_BLOCK_M, &tmS, &full_bar[stage], m_tile * F8_BLOCK_M, kb);
          if (++stage == F8_STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ------------------------------- consumers: MMA + promotion + epilogue -------------------------------
    setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;
    const int q4 = lane >> 2, c2 = 2 * (lane & 3);   // fragment: rows q4 / q4 + 8 of the warp's 16, columns 8g + c2, +1
    const int r_lo = wg * 64 + (warp & 3) * 16 + q4;  // tile row of this thread's first fragment row
    int stage = 0;
    uint32_t phase = 0;
    float acc[64], accp[64];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int m_tile, n_tile;
      f8_tile_coords(tile, p.num_m_tiles, p.num_n_tiles, m_tile, n_tile);
#pragma unroll
      for (int i = 0; i < 64; ++i) accp[i] = 0.f;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * 2 * F8_TILE_BYTES);
        const uint64_t ad = make_smem_desc_sw128(sa + wg * 64 * 128, 16, 1024);
        const uint64_t bd = make_smem_desc_sw128(sa + F8_TILE_BYTES, 16, 1024);
        fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < F8_BLOCK_K / 32; ++k) wgmma_e4m3_n128(acc, ad + 2 * k, bd + 2 * k, k == 0 ? 0u : 1u);   // 32 B per k-step
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(acc);
        const float s_lo = sscale[stage * F8_BLOCK_M + r_lo];
        const float s_hi = sscale[stage * F8_BLOCK_M + r_lo + 8];
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == F8_STAGES) {
          stage = 0;
          phase ^= 1;
        }
#pragma unroll
        for (int g = 0; g < 16; ++g) {   // promotion: one fp32 FMA per element and k-group
          accp[4 * g + 0] = fmaf(s_lo, acc[4 * g + 0], accp[4 * g + 0]);
          accp[4 * g + 1] = fmaf(s_lo, acc[4 * g + 1], accp[4 * g + 1]);
          accp[4 * g + 2] = fmaf(s_hi, acc[4 * g + 2], accp[4 * g + 2]);
          accp[4 * g + 3] = fmaf(s_hi, acc[4 * g + 3], accp[4 * g + 3]);
        }
      }

      // ---- epilogue: v = accp * s_w[n] + bias[n], straight from the fragment (4 lanes write 8 adjacent columns of a row)
      const int n0 = n_tile * F8_BLOCK_N;
      const int row_lo = m_tile * F8_BLOCK_M + r_lo, row_hi = row_lo + 8;
      int tok_lo = 0, tok_hi = 0;
      if (EPI == YB_EPI_GATE_RES && p.gate != nullptr && p.tok_idx != nullptr) {
        if (row_lo < p.M) tok_lo = p.tok_idx[row_lo];
        if (row_hi < p.M) tok_hi = p.tok_idx[row_hi];
      }
#pragma unroll
      for (int g = 0; g < 16; ++g) {
        const int col = n0 + 8 * g + c2;
        const float2 sw = __ldg(reinterpret_cast<const float2*>(p.b_scale + col));
        float2 b = make_float2(0.f, 0.f);
        if (p.bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
        accp[4 * g + 0] = accp[4 * g + 0] * sw.x + b.x;
        accp[4 * g + 1] = accp[4 * g + 1] * sw.y + b.y;
        accp[4 * g + 2] = accp[4 * g + 2] * sw.x + b.x;
        accp[4 * g + 3] = accp[4 * g + 3] * sw.y + b.y;
      }
      if (EPI == YB_EPI_GELU_FP8) {
        // gelu_tanh, then the 1x128 quantisation of each row segment: this tile's 128 columns ARE one group
        float m_lo = 0.f, m_hi = 0.f;
#pragma unroll
        for (int i = 0; i < 64; ++i) accp[i] = gelu_tanh(accp[i]);
#pragma unroll
        for (int g = 0; g < 16; ++g) {
          m_lo = fmaxf(m_lo, fmaxf(fabsf(accp[4 * g]), fabsf(accp[4 * g + 1])));
          m_hi = fmaxf(m_hi, fmaxf(fabsf(accp[4 * g + 2]), fabsf(accp[4 * g + 3])));
        }
        m_lo = fmaxf(m_lo, __shfl_xor_sync(0xffffffffu, m_lo, 1));
        m_lo = fmaxf(m_lo, __shfl_xor_sync(0xffffffffu, m_lo, 2));
        m_hi = fmaxf(m_hi, __shfl_xor_sync(0xffffffffu, m_hi, 1));
        m_hi = fmaxf(m_hi, __shfl_xor_sync(0xffffffffu, m_hi, 2));
        float inv_lo, sc_lo, inv_hi, sc_hi;
        group_scale(m_lo, inv_lo, sc_lo);
        group_scale(m_hi, inv_hi, sc_hi);
        uint8_t* o8 = reinterpret_cast<uint8_t*>(p.out);
#pragma unroll
        for (int g = 0; g < 16; ++g) {
          const int col = n0 + 8 * g + c2;
          if (row_lo < p.M)
            *reinterpret_cast<uint16_t*>(o8 + static_cast<long long>(row_lo) * p.ldo + col) =
                cvt_e4m3x2(accp[4 * g] * inv_lo, accp[4 * g + 1] * inv_lo);
          if (row_hi < p.M)
            *reinterpret_cast<uint16_t*>(o8 + static_cast<long long>(row_hi) * p.ldo + col) =
                cvt_e4m3x2(accp[4 * g + 2] * inv_hi, accp[4 * g + 3] * inv_hi);
        }
        if ((lane & 3) == 0) {
          float* srow = p.out_scale + static_cast<long long>(n0 / 128) * p.ldos;
          if (row_lo < p.M) srow[row_lo] = sc_lo;
          if (row_hi < p.M) srow[row_hi] = sc_hi;
        }
      } else if (EPI == YB_EPI_BF16) {
        __nv_bfloat16* ob = reinterpret_cast<__nv_bfloat16*>(p.out);
#pragma unroll
        for (int g = 0; g < 16; ++g) {
          const int col = n0 + 8 * g + c2;
          if (row_lo < p.M)
            *reinterpret_cast<uint32_t*>(ob + static_cast<long long>(row_lo) * p.ldo + col) = pack_bf16x2(accp[4 * g], accp[4 * g + 1]);
          if (row_hi < p.M)
            *reinterpret_cast<uint32_t*>(ob + static_cast<long long>(row_hi) * p.ldo + col) =
                pack_bf16x2(accp[4 * g + 2], accp[4 * g + 3]);
        }
      } else {   // YB_EPI_F32 / YB_EPI_GATE_RES: fp32 rows
        float* of = reinterpret_cast<float*>(p.out);
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int row = half ? row_hi : row_lo;
          if (row >= p.M) continue;
          const long long tok = half ? tok_hi : tok_lo;
          float* orow = of + static_cast<long long>(row) * p.ldo;
#pragma unroll
          for (int g = 0; g < 16; ++g) {
            const int col = n0 + 8 * g + c2;
            float2 v = make_float2(accp[4 * g + 2 * half], accp[4 * g + 2 * half + 1]);
            float2* o2 = reinterpret_cast<float2*>(orow + col);
            if (EPI == YB_EPI_GATE_RES) {
              float2 gt = make_float2(1.f, 1.f);
              if (p.gate) gt = __ldg(reinterpret_cast<const float2*>(p.gate + tok * p.gate_ld + col));
              float2 x = *o2;
              x.x += v.x * gt.x;
              x.y += v.y * gt.y;
              *o2 = x;
            } else {
              *o2 = v;
            }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm (+ adaLN modulate or the affine norm3) -> e4m3 + 1x128 scales. The fp32 arithmetic is that of
// ln_modulate_warp_kernel<NV, true, ADA> (elementwise.cu), so the quantised values are those of the f32 output of yb_ln_modulate.
// Lane l holds float4 l + 32 i of the row: float4 block i (32 lanes x 4) is scale group i.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float f8_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float4 f8_ldg_f4_ordered(const float* p) {
  float4 v;
  asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}

// quantise one float4 with the group's inv and store its 4 bytes
__device__ __forceinline__ void store_e4m3x4(uint8_t* dst, float4 y, float inv) {
  const uint32_t lo = cvt_e4m3x2(y.x * inv, y.y * inv), hi = cvt_e4m3x2(y.z * inv, y.w * inv);
  *reinterpret_cast<uint32_t*>(dst) = lo | (hi << 16);
}

template <int NV, bool ADA>
__global__ void __launch_bounds__(256)
ln_modulate_fp8_kernel(const float* __restrict__ x, long long ldx, uint8_t* __restrict__ out, long long ldo,
                       float* __restrict__ out_scale, long long lds, const float* __restrict__ mul,
                       const float* __restrict__ add, long long mod_ld, const int* __restrict__ tok_idx, int L, float eps) {
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
  const float mean = f8_warp_sum(s) * (1.0f / C);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = rsqrtf(f8_warp_sum(q) * (1.0f / C) + eps);
  const long long u = (ADA && tok_idx) ? tok_idx[row] : 0;
  const float* mp = mul ? mul + u * mod_ld + lane * 4 : nullptr;
  const float* ap = add ? add + u * mod_ld + lane * 4 : nullptr;
  uint8_t* orow = out + static_cast<long long>(row) * ldo;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    float4 cm = make_float4(0.f, 0.f, 0.f, 0.f), ca = cm;
    if (mp) cm = f8_ldg_f4_ordered(mp + i * 128);
    if (ap) ca = f8_ldg_f4_ordered(ap + i * 128);
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
    const float amax = f8_warp_max(amax4(y.x, y.y, y.z, y.w));
    float inv, scale;
    group_scale(amax, inv, scale);
    store_e4m3x4(orow + (lane + i * 32) * 4, y, inv);
    if (lane == 0) out_scale[static_cast<long long>(i) * lds + row] = scale;
  }
}

// bf16 rows -> e4m3 + 1x128 scales: one warp per row, one 128-column group per step (lane l: columns 4l .. 4l + 3)
__global__ void __launch_bounds__(256)
quant_rows_fp8_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, uint8_t* __restrict__ out, long long ldo,
                      float* __restrict__ out_scale, long long lds, int M, int groups) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const __nv_bfloat16* xr = x + static_cast<long long>(row) * ldx + lane * 4;
  uint8_t* orow = out + static_cast<long long>(row) * ldo + lane * 4;
  for (int g = 0; g < groups; ++g) {
    const uint2 raw = __ldg(reinterpret_cast<const uint2*>(xr + g * 128));
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.x));
    const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&raw.y));
    const float4 y = make_float4(a.x, a.y, b.x, b.y);
    const float amax = f8_warp_max(amax4(y.x, y.y, y.z, y.w));
    float inv, scale;
    group_scale(amax, inv, scale);
    store_e4m3x4(orow + g * 128, y, inv);
    if (lane == 0) out_scale[static_cast<long long>(g) * lds + row] = scale;
  }
}

// 2-D tensor maps of the fp8 GEMM: e4m3 operand [rows, cols] (row stride ld bytes, 128B swizzle, box 128 x 128) and the f32
// scale table [groups, lds] read as [groups][M] (box {128 rows of one group}, no swizzle; rows >= M are zero fill)
static int make_tmap_e4m3(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint64_t ld) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return YB_ERR_NO_DRIVER;
  if ((reinterpret_cast<uintptr_t>(base) & 0xF) || (ld & 0xF)) return YB_ERR_ALIGNMENT;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld};
  cuuint32_t box[2] = {F8_BLOCK_K, 128};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? YB_OK : YB_ERR_TENSORMAP;
}

static int make_tmap_scales(CUtensorMap* tm, const void* base, uint64_t M, uint64_t groups, uint64_t lds) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return YB_ERR_NO_DRIVER;
  if ((reinterpret_cast<uintptr_t>(base) & 0xF) || (lds % 4)) return YB_ERR_ALIGNMENT;
  cuuint64_t gdim[2] = {M, groups};
  cuuint64_t gstride[1] = {lds * 4};
  cuuint32_t box[2] = {F8_BLOCK_M, 1};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? YB_OK : YB_ERR_TENSORMAP;
}

template <int EPI>
static int launch_gemm_fp8(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmS, const Fp8Params& p,
                           cudaStream_t stream) {
  static bool attr_set[kMaxDevices] = {};
  if (int rc = ensure_dynamic_smem(gemm_fp8_kernel<EPI>, F8_SMEM_BYTES, attr_set, "gemm_fp8")) return rc;
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  const int grid = tiles < sm_count() ? tiles : sm_count();
  gemm_fp8_kernel<EPI><<<grid, F8_THREADS, F8_SMEM_BYTES, stream>>>(tmA, tmB, tmS, p);
  return check_launch("gemm_fp8");
}

}  // namespace yb

extern "C" int yb_gemm_fp8(const yb_gemm_fp8_args* a, void* stream_) {
  using namespace yb;
  if (!a || a->struct_bytes != sizeof(yb_gemm_fp8_args)) return YB_ERR_ARG;
  if (!a->A || !a->a_scale || !a->B || !a->b_scale || !a->out) return YB_ERR_ARG;
  if (a->M <= 0 || a->N <= 0 || a->K <= 0) return YB_ERR_ARG;
  const int epi = a->epilogue;
  if (epi != YB_EPI_BF16 && epi != YB_EPI_F32 && epi != YB_EPI_GATE_RES && epi != YB_EPI_GELU_FP8) return YB_ERR_ARG;
  if (a->block_n != 0 && a->block_n != F8_BLOCK_N) return YB_ERR_ARG;
  if (a->N % F8_BLOCK_N != 0 || a->K % F8_BLOCK_K != 0) return YB_ERR_SHAPE;
  if (a->lds < a->M || (epi == YB_EPI_GELU_FP8 && (!a->out_scale || a->ldos < a->M))) return YB_ERR_ARG;
  const long long ldo_mult = epi == YB_EPI_BF16 ? 8 : epi == YB_EPI_GELU_FP8 ? 16 : 4;
  if ((a->ldo % ldo_mult) || (reinterpret_cast<uintptr_t>(a->out) & 0xF) || (a->lds % 4) ||
      (reinterpret_cast<uintptr_t>(a->b_scale) & 0x7) || (reinterpret_cast<uintptr_t>(a->bias) & 0x7) ||
      (epi == YB_EPI_GELU_FP8 && ((a->ldos % 4) || (reinterpret_cast<uintptr_t>(a->out_scale) & 0xF))))
    return YB_ERR_ALIGNMENT;
  if (epi == YB_EPI_GATE_RES && a->gate && ((a->gate_ld % 2) || (reinterpret_cast<uintptr_t>(a->gate) & 0x7))) return YB_ERR_ALIGNMENT;
  CUtensorMap tmA, tmB, tmS;
  int rc = make_tmap_e4m3(&tmA, a->A, a->M, a->K, a->lda);
  if (rc) return rc;
  rc = make_tmap_e4m3(&tmB, a->B, a->N, a->K, a->ldb);
  if (rc) return rc;
  rc = make_tmap_scales(&tmS, a->a_scale, a->M, a->K / F8_BLOCK_K, a->lds);
  if (rc) return rc;
  Fp8Params p;
  p.M = a->M;
  p.N = a->N;
  p.K = a->K;
  p.num_m_tiles = (a->M + F8_BLOCK_M - 1) / F8_BLOCK_M;
  p.num_n_tiles = a->N / F8_BLOCK_N;
  p.b_scale = static_cast<const float*>(a->b_scale);
  p.bias = static_cast<const float*>(a->bias);
  p.out = a->out;
  p.ldo = a->ldo;
  p.out_scale = static_cast<float*>(a->out_scale);
  p.ldos = a->ldos;
  p.gate = static_cast<const float*>(a->gate);
  p.gate_ld = a->gate_ld;
  p.tok_idx = static_cast<const int*>(a->tok_idx);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  switch (epi) {
    case YB_EPI_BF16: return launch_gemm_fp8<YB_EPI_BF16>(tmA, tmB, tmS, p, stream);
    case YB_EPI_F32: return launch_gemm_fp8<YB_EPI_F32>(tmA, tmB, tmS, p, stream);
    case YB_EPI_GATE_RES: return launch_gemm_fp8<YB_EPI_GATE_RES>(tmA, tmB, tmS, p, stream);
    default: return launch_gemm_fp8<YB_EPI_GELU_FP8>(tmA, tmB, tmS, p, stream);
  }
}

extern "C" int yb_ln_modulate_fp8(const void* x, long long ldx, void* out, long long ldo, void* out_scale, long long lds,
                                  const void* scale, const void* shift, long long mod_ld, const void* tok_idx, const void* weight,
                                  const void* lnbias, int L, int C, float eps, void* stream_) {
  using namespace yb;
  if (!x || !out || !out_scale || L <= 0 || C <= 0 || lds < L) return YB_ERR_ARG;
  const bool ada = scale || shift, affine = weight || lnbias;
  if (ada && affine) return YB_ERR_ARG;
  if ((ldx % 4) || (ldo % 16) || (mod_ld % 4) || (lds % 4) || (reinterpret_cast<uintptr_t>(x) & 0xF) ||
      (reinterpret_cast<uintptr_t>(out) & 0xF) || (reinterpret_cast<uintptr_t>(out_scale) & 0x3))
    return YB_ERR_ALIGNMENT;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  const float* mul = static_cast<const float*>(affine ? weight : scale);
  const float* add = static_cast<const float*>(affine ? lnbias : shift);
#define YB_LN8(NV)                                                                                                      \
  if (C == (NV) * 128) {                                                                                                \
    if (affine)                                                                                                         \
      ln_modulate_fp8_kernel<NV, false><<<(L + 7) / 8, 256, 0, s>>>(static_cast<const float*>(x), ldx,                  \
          static_cast<uint8_t*>(out), ldo, static_cast<float*>(out_scale), lds, mul, add, mod_ld, nullptr, L, eps);     \
    else                                                                                                                \
      ln_modulate_fp8_kernel<NV, true><<<(L + 7) / 8, 256, 0, s>>>(static_cast<const float*>(x), ldx,                   \
          static_cast<uint8_t*>(out), ldo, static_cast<float*>(out_scale), lds, mul, add, mod_ld,                       \
          static_cast<const int*>(tok_idx), L, eps);                                                                    \
    return check_launch("ln_modulate_fp8");                                                                             \
  }
  YB_LN8(24)
  YB_LN8(40)
  YB_LN8(8)
  YB_LN8(2)
#undef YB_LN8
  return YB_ERR_SHAPE;
}

extern "C" int yb_quant_rows_fp8(const void* x, long long ldx, void* out, long long ldo, void* out_scale, long long lds, int M, int K,
                                 void* stream_) {
  using namespace yb;
  if (!x || !out || !out_scale || M <= 0 || K <= 0 || lds < M) return YB_ERR_ARG;
  if (K % 128 != 0) return YB_ERR_SHAPE;
  if ((ldx % 8) || (ldo % 16) || (lds % 4) || (reinterpret_cast<uintptr_t>(x) & 0xF) || (reinterpret_cast<uintptr_t>(out) & 0xF) ||
      (reinterpret_cast<uintptr_t>(out_scale) & 0x3))
    return YB_ERR_ALIGNMENT;
  quant_rows_fp8_kernel<<<(M + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __nv_bfloat16*>(x), ldx, static_cast<uint8_t*>(out), ldo, static_cast<float*>(out_scale), lds, M, K / 128);
  return check_launch("quant_rows_fp8");
}
