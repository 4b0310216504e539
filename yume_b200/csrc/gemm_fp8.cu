// gemm_fp8.cu — the FP8 (e4m3) block-scaled wgmma kernel on sm_90a (H100) with per-group promotion, and the two kernels that
// produce the DiT GEMMs' 1x128-quantised activations (LayerNorm + modulate, and bf16 rows). The kernel has two modes:
//   CONV = 0   the DiT block GEMMs; numerics and constraints: include/yume_b200_fp8.h
//   CONV = 1   the implicit-GEMM causal conv of the Wan2.2 VAE decode; numerics and constraints: include/yume_b200_fp8_vae.h. Its
//              A operand is that of the bf16 conv (gemm.cu): a 4-D TMA box of 128 output voxels per tap, out-of-bounds zero fill
// Structure follows gemm.cu (persistent, warp-specialised, TMA ring). One k-group (GEMM: 128 columns of K; conv: one 128-channel
// group of one tap) per ring stage:
//   warp 0               producer: A tile 128 x 128 e4m3, B tile 128 x 128 e4m3 (128B swizzle: one 128-byte swizzle row is
//                        exactly one scale group) and the 128 A-scales of that k-group (512 B) into stage s of the ring.
//                        GEMM: one thread issues the three TMA loads. Conv: lane 0 issues the two tiles and all 32 lanes gather
//                        the scales of the tap-shifted voxels (0 outside the input); the stage's full barrier counts the 32 lane
//                        arrivals and the TMA bytes
//   warpgroups 1-2       consumers, rows [64 * (wg - 1), +64): per k-group 4 x wgmma m64n128k32 into a fresh accumulator, wait,
//                        then promotion acc_p += s_a[row] * acc (fp32 FMA); epilogue straight from the fragment registers
// The conv's scales go through the producer's lanes, not TMA: a TMA box of fp32 needs a 16-byte inner extent, and narrow boxes
// (TW < 4) do occur at the small levels.
#include <type_traits>

#include "yb_host.h"
#include "../../include/yume_b200_fp8.h"
#include "../../include/yume_b200_fp8_vae.h"
#include "../../include/yume_b200_fp8_sp.h"
#include "yb_ptx.cuh"

namespace yb {

constexpr int F8_BLOCK_M = 128;                              // GEMM: rows; conv: output voxels (TT x TH x TW)
constexpr int F8_BLOCK_N = 128;
constexpr int F8_BLOCK_K = 128;                              // 128 e4m3 = 128 B = one swizzle row = one scale group
constexpr int F8_THREADS = 384;
constexpr int F8_TILE_BYTES = 128 * 128;                     // one operand tile
constexpr int F8_STAGES = 6;
constexpr int F8_SCALE_BYTES = F8_BLOCK_M * 4;
constexpr int F8_SMEM_BYTES = 1024 + F8_STAGES * (2 * F8_TILE_BYTES + F8_SCALE_BYTES) + 256;

// |x| for the group maximum: a NaN element does not take part (fmaxf returns the other operand)
__device__ __forceinline__ float amax4(float a, float b, float c, float d) {
  return fmaxf(fmaxf(fabsf(a), fabsf(b)), fmaxf(fabsf(c), fabsf(d)));
}

__device__ __forceinline__ float f8_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Parameters of the two modes. The fields both modes use have the same names, so the shared code reads either struct. They stay
// two structs: one holding both modes' fields would pass 128 bytes, and past that nvcc reads the kernel parameters through a
// pointer in registers instead of from the constant bank.
struct GemmFp8Params {
  int M, N, K, num_m_tiles, num_n_tiles;
  const float* b_scale;   // [N] per output channel
  const float* bias;      // [N] or null
  void* out;
  long long ldo;
  float* out_scale;
  long long ldos;
  const float* gate;
  long long gate_ld;
  const int* tok_idx;
};

struct ConvFp8Params {
  const float* x_scale;   // [inT, groups, H, W]
  const float* b_scale;   // [Cout] per output channel
  const float* bias;      // [Cout] or null
  __nv_bfloat16* out;
  long long ldo;
  const __nv_bfloat16* res;
  long long res_ld;
  int inT, H, W, groups;  // input extents (history frames included) and Cp / 128
  int T;                  // output frames
  int taps;               // kt * 9: the spatial taps are always 3 x 3
  int off_t, off_h, off_w;
  int TW, TH, TT, tiles_w, tiles_h;
  int lg_tw, lg_twh;      // log2 TW, log2 (TW * TH)
  int num_m_tiles, num_n_tiles;
};

template <int CONV>
using Fp8Params = std::conditional_t<CONV != 0, ConvFp8Params, GemmFp8Params>;

// conv: m tile -> origin (t0, h0, w0) of its TT x TH x TW output box
__device__ __forceinline__ void conv_box_origin(const ConvFp8Params& p, int mt, int& t0, int& h0, int& w0) {
  const int per_t = p.tiles_h * p.tiles_w;
  const int it = mt / per_t;
  const int rem = mt - it * per_t;
  const int ih = rem / p.tiles_w;
  t0 = it * p.TT;
  h0 = ih * p.TH;
  w0 = (rem - ih * p.tiles_w) * p.TW;
}

template <int EPI, int CONV>
__global__ void __launch_bounds__(F8_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmS, const Fp8Params<CONV> p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* sscale = reinterpret_cast<float*>(smem + F8_STAGES * 2 * F8_TILE_BYTES);   // [stage][128]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sscale + F8_STAGES * F8_BLOCK_M);
  uint64_t* empty_bar = full_bar + F8_STAGES;

  const int warp = threadIdx.x >> 5;
  // lane, tiles of the launch and k-groups per tile: formed once here for the GEMM, and by each role after its setmaxnreg for the
  // conv, whose producer has 48 registers (held across the setmaxnreg, the values spill)
  int lane, num_tiles, num_kb;
  auto role_init = [&]() {
    lane = threadIdx.x & 31;
    num_tiles = p.num_m_tiles * p.num_n_tiles;
    if constexpr (CONV) num_kb = p.taps * p.groups;
    else num_kb = p.K / F8_BLOCK_K;
  };
  if constexpr (!CONV) role_init();

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (!CONV) tma_prefetch_desc(&tmS);
    for (int i = 0; i < F8_STAGES; ++i) {
      mbar_init(&full_bar[i], CONV ? 32 : 1);   // conv: the 32 producer lanes (lane 0's arrival also brings the TMA byte count)
      mbar_init(&empty_bar[i], 8);               // the 8 consumer warps
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    if constexpr (CONV) {
      setmaxnreg_dec<48>();   // 128 x 48 + 256 x 224 <= 384 x 168, the registers the launch holds
      if (warp == 0) {
        // ------------------------------- conv producer (whole warp) -------------------------------
        role_init();
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
          int m_tile, n_tile, t0, h0, w0;
          tile_coords(tile, p.num_m_tiles, p.num_n_tiles, m_tile, n_tile);
          conv_box_origin(p, m_tile, t0, h0, w0);
          // the scales of k-group kb are fetched one k-group ahead, so their latency hides behind the slot wait and the TMA
          // issue. Box row r = (tt * TH + th) * TW + tw (TW, TH powers of two); the tap-shifted input voxel of row lane + 32 i
          // is recomputed per fetch: the producer has 48 registers
          auto fetch = [&](int kb, float (&s)[4]) {
            const int tap = kb / p.groups, g = kb - tap * p.groups;
            const int dt = tap / 9, dh = (tap / 3) % 3, dw = tap % 3;   // kh = kw = 3
            const int tb = t0 + dt - p.off_t, hb = h0 + dh - p.off_h, wb = w0 + dw - p.off_w;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int r = lane + 32 * i;
              const int t = tb + (r >> p.lg_twh), h = hb + ((r >> p.lg_tw) & (p.TH - 1)), w = wb + (r & (p.TW - 1));
              const bool in = static_cast<unsigned>(t) < static_cast<unsigned>(p.inT) &&
                              static_cast<unsigned>(h) < static_cast<unsigned>(p.H) && static_cast<unsigned>(w) < static_cast<unsigned>(p.W);
              s[i] = in ? __ldg(p.x_scale + ((t * p.groups + g) * p.H + h) * p.W + w) : 0.f;   // < 2^31 elements (host check)
            }
          };
          float cur[4];
          fetch(0, cur);
          for (int kb = 0; kb < num_kb; ++kb) {
            float nxt[4] = {0.f, 0.f, 0.f, 0.f};
            if (kb + 1 < num_kb) fetch(kb + 1, nxt);
            mbar_wait(&empty_bar[stage], phase ^ 1);
            float* ss = sscale + stage * F8_BLOCK_M;
#pragma unroll
            for (int i = 0; i < 4; ++i) ss[lane + 32 * i] = cur[i];
            if (lane == 0) {
              const int tap = kb / p.groups, g = kb - tap * p.groups;
              const int dt = tap / 9, dh = (tap / 3) % 3, dw = tap % 3;
              uint8_t* sa = smem + stage * 2 * F8_TILE_BYTES;
              mbar_arrive_expect_tx(&full_bar[stage], 2 * F8_TILE_BYTES);
              tma_load_4d(sa, &tmA, &full_bar[stage], g * F8_BLOCK_K, w0 + dw - p.off_w, h0 + dh - p.off_h, t0 + dt - p.off_t);
              tma_load_2d(sa + F8_TILE_BYTES, &tmB, &full_bar[stage], kb * F8_BLOCK_K, n_tile * F8_BLOCK_N);
            } else {
              mbar_arrive(&full_bar[stage]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) cur[i] = nxt[i];
            if (++stage == F8_STAGES) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      }
    } else {
      setmaxnreg_dec<40>();
      if (warp == 0 && lane == 0) {
        // ------------------------------- GEMM TMA producer (one thread) -------------------------------
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
          int m_tile, n_tile;
          tile_coords(tile, p.num_m_tiles, p.num_n_tiles, m_tile, n_tile);
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
    }
  } else {
    // ------------------------------- consumers: MMA + promotion + epilogue -------------------------------
    if constexpr (CONV) setmaxnreg_inc<224>();
    else setmaxnreg_inc<232>();
    if constexpr (CONV) role_init();
    const int wg = (warp >> 2) - 1;
    const int q4 = lane >> 2, c2 = 2 * (lane & 3);   // fragment: rows q4 / q4 + 8 of the warp's 16, columns 8g + c2, +1
    const int r_lo = wg * 64 + (warp & 3) * 16 + q4;  // tile row of this thread's first fragment row
    int stage = 0;
    uint32_t phase = 0;
    float acc[64], accp[64];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int m_tile, n_tile;
      tile_coords(tile, p.num_m_tiles, p.num_n_tiles, m_tile, n_tile);
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
        for (int k = 0; k < F8_BLOCK_K / 32; ++k) wgmma_ss_e4m3(acc, ad + 2 * k, bd + 2 * k, k == 0 ? 0u : 1u);   // 32 B per k-step
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

      if constexpr (CONV) {
        // ---- epilogue: v = accp * s_w[n] + bias[n] (+ res), bf16, straight from the fragment; rows outside the output are skipped
        int t0, h0, w0;
        conv_box_origin(p, m_tile, t0, h0, w0);
        long long orow[2];
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int r = r_lo + 8 * half;
          const int t = t0 + (r >> p.lg_twh), h = h0 + ((r >> p.lg_tw) & (p.TH - 1)), w = w0 + (r & (p.TW - 1));
          orow[half] = (t < p.T && h < p.H && w < p.W) ? (static_cast<long long>(t) * p.H + h) * p.W + w : -1;
        }
        const int n0 = n_tile * F8_BLOCK_N;
#pragma unroll
        for (int g = 0; g < 16; ++g) {
          const int col = n0 + 8 * g + c2;
          const float2 sw = __ldg(reinterpret_cast<const float2*>(p.b_scale + col));
          float2 b = make_float2(0.f, 0.f);
          if (p.bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            if (orow[half] < 0) continue;
            float vx = accp[4 * g + 2 * half] * sw.x + b.x;
            float vy = accp[4 * g + 2 * half + 1] * sw.y + b.y;
            if (EPI == YB_EPI_RES_BF16) {
              const float2 rv = __bfloat1622float2(
                  *reinterpret_cast<const __nv_bfloat162*>(p.res + orow[half] * p.res_ld + col));
              vx += rv.x;
              vy += rv.y;
            }
            *reinterpret_cast<uint32_t*>(p.out + orow[half] * p.ldo + col) = pack_bf16x2(vx, vy);
          }
        }
      } else {
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
  *reinterpret_cast<uint32_t*>(dst) = cvt_e4m3x4(y.x * inv, y.y * inv, y.z * inv, y.w * inv);
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

// quant_rows_fp8_kernel over a K-split source (yb_quant_rows_fp8_split): group g of row m lies in chunk (g * 128) / split, at
// column (g * 128) % split of that chunk's row m; the arithmetic per group is quant_rows_fp8_kernel's
__global__ void __launch_bounds__(256)
quant_rows_fp8_split_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, int split, long long split_stride,
                            uint8_t* __restrict__ out, long long ldo, float* __restrict__ out_scale, long long lds, int M,
                            int groups) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const __nv_bfloat16* xr = x + static_cast<long long>(row) * ldx + lane * 4;
  uint8_t* orow = out + static_cast<long long>(row) * ldo + lane * 4;
  const int per_chunk = split >> 7;
  for (int g = 0; g < groups; ++g) {
    const int chunk = g / per_chunk;
    const uint2 raw = __ldg(reinterpret_cast<const uint2*>(xr + chunk * split_stride + (g - chunk * per_chunk) * 128));
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

// 4-D e4m3 tensor map over a dense channels-last volume [T, H, W, C] (C bytes per voxel), box {128 channels, bw, bh, bt}, 128-byte
// swizzle, out-of-bounds voxels read as zeros
static int make_tmap_e4m3_4d(CUtensorMap* tm, const void* base, uint64_t T, uint64_t H, uint64_t W, uint64_t C, uint32_t bt,
                             uint32_t bh, uint32_t bw) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return YB_ERR_NO_DRIVER;
  if ((reinterpret_cast<uintptr_t>(base) & 0xF) || (C & 0xF)) return YB_ERR_ALIGNMENT;
  cuuint64_t gdim[4] = {C, W, H, T};
  cuuint64_t gstride[3] = {C, W * C, H * W * C};
  cuuint32_t box[4] = {F8_BLOCK_K, bw, bh, bt};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  if (bw > 256 || bh > 256 || bt > 256) return YB_ERR_SHAPE;
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? YB_OK : YB_ERR_TENSORMAP;
}

// tmS: the GEMM's A-scale map (the conv's producer gathers its scales instead)
template <int EPI, int CONV>
static int launch_gemm_fp8(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmS, const Fp8Params<CONV>& p,
                           cudaStream_t stream) {
  const char* what = CONV ? "conv3d_fp8" : "gemm_fp8";
  static bool attr_set[kMaxDevices] = {};
  if (int rc = ensure_dynamic_smem(gemm_fp8_kernel<EPI, CONV>, F8_SMEM_BYTES, attr_set, what)) return rc;
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  const int grid = tiles < sm_count() ? tiles : sm_count();
  gemm_fp8_kernel<EPI, CONV><<<grid, F8_THREADS, F8_SMEM_BYTES, stream>>>(tmA, tmB, tmS, p);
  return check_launch(what);
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
  int rc = make_tmap_e4m3_2d(&tmA, a->A, a->M, a->K, a->lda);
  if (rc) return rc;
  rc = make_tmap_e4m3_2d(&tmB, a->B, a->N, a->K, a->ldb);
  if (rc) return rc;
  rc = make_tmap_f32_scales(&tmS, a->a_scale, a->M, a->K / F8_BLOCK_K, a->lds);
  if (rc) return rc;
  GemmFp8Params p = {};
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
    case YB_EPI_BF16: return launch_gemm_fp8<YB_EPI_BF16, 0>(tmA, tmB, tmS, p, stream);
    case YB_EPI_F32: return launch_gemm_fp8<YB_EPI_F32, 0>(tmA, tmB, tmS, p, stream);
    case YB_EPI_GATE_RES: return launch_gemm_fp8<YB_EPI_GATE_RES, 0>(tmA, tmB, tmS, p, stream);
    default: return launch_gemm_fp8<YB_EPI_GELU_FP8, 0>(tmA, tmB, tmS, p, stream);
  }
}

extern "C" int yb_conv3d_fp8(const yb_conv3d_fp8_args* a, void* stream_) {
  using namespace yb;
  if (!a || a->struct_bytes != sizeof(yb_conv3d_fp8_args)) return YB_ERR_ARG;
  if (!a->x || !a->x_scale || !a->w || !a->w_scale || !a->out) return YB_ERR_ARG;
  if (a->T <= 0 || a->H <= 0 || a->W <= 0 || a->Cp <= 0 || a->Cout <= 0) return YB_ERR_ARG;
  if (a->epilogue != YB_EPI_BF16 && a->epilogue != YB_EPI_RES_BF16) return YB_ERR_ARG;
  if (a->epilogue == YB_EPI_RES_BF16 && !a->res) return YB_ERR_ARG;
  if (a->Cp % 128 != 0 || a->Cout % 128 != 0) return YB_ERR_SHAPE;
  if ((a->kt != 1 && a->kt != 3) || a->kh != 3 || a->kw != 3) return YB_ERR_SHAPE;
  if (a->t_hist != 0 && a->t_hist != a->kt - 1) return YB_ERR_ARG;
  if ((a->ldo % 8) || (reinterpret_cast<uintptr_t>(a->out) & 0xF) || (reinterpret_cast<uintptr_t>(a->x_scale) & 0x3) ||
      (reinterpret_cast<uintptr_t>(a->w_scale) & 0x7) || (reinterpret_cast<uintptr_t>(a->bias) & 0x7) ||
      (a->epilogue == YB_EPI_RES_BF16 && ((a->res_ld % 2) || (reinterpret_cast<uintptr_t>(a->res) & 0x3))))
    return YB_ERR_ALIGNMENT;
  const long long inT = static_cast<long long>(a->T) + a->t_hist;
  if (inT * a->H * a->W * (a->Cp / 128) > 0x7fffffffLL) return YB_ERR_SHAPE;   // 32-bit scale and voxel indices in the kernel
  int plan[4];
  if (int rc = yb_conv3d_plan(a->T, a->H, a->W, a->Cout, a->kw, 1, plan)) return rc;   // the bf16 conv's box rule, kw not fused
  ConvFp8Params p = {};
  p.TW = plan[0];
  p.TH = plan[1];
  p.TT = plan[2];
  p.x_scale = static_cast<const float*>(a->x_scale);
  p.b_scale = static_cast<const float*>(a->w_scale);
  p.bias = static_cast<const float*>(a->bias);
  p.out = static_cast<__nv_bfloat16*>(a->out);
  p.ldo = a->ldo;
  p.res = static_cast<const __nv_bfloat16*>(a->res);
  p.res_ld = a->res_ld;
  p.inT = static_cast<int>(inT);
  p.H = a->H;
  p.W = a->W;
  p.groups = a->Cp / 128;
  p.T = a->T;
  p.lg_tw = __builtin_ctz(p.TW);
  p.lg_twh = __builtin_ctz(p.TW * p.TH);
  p.taps = a->kt * a->kh * a->kw;
  p.off_t = a->kt - 1 - a->t_hist;   // output frame t reads input frames t + t_hist - (kt - 1) + dt of the map
  p.off_h = a->kh / 2;
  p.off_w = a->kw / 2;
  p.tiles_w = (a->W + p.TW - 1) / p.TW;
  p.tiles_h = (a->H + p.TH - 1) / p.TH;
  p.num_m_tiles = ((a->T + p.TT - 1) / p.TT) * p.tiles_h * p.tiles_w;
  p.num_n_tiles = a->Cout / F8_BLOCK_N;
  CUtensorMap tmA, tmB, tmS = {};
  int rc = make_tmap_e4m3_4d(&tmA, a->x, inT, a->H, a->W, a->Cp, p.TT, p.TH, p.TW);
  if (rc) return rc;
  const uint64_t K = static_cast<uint64_t>(p.taps) * a->Cp;
  rc = make_tmap_e4m3_2d(&tmB, a->w, a->Cout, K, K);
  if (rc) return rc;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (a->epilogue == YB_EPI_RES_BF16) return launch_gemm_fp8<YB_EPI_RES_BF16, 1>(tmA, tmB, tmS, p, stream);
  return launch_gemm_fp8<YB_EPI_BF16, 1>(tmA, tmB, tmS, p, stream);
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

extern "C" int yb_quant_rows_fp8_split(const void* x, long long ldx, int split, long long split_stride, void* out, long long ldo,
                                       void* out_scale, long long lds, int M, int K, void* stream_) {
  using namespace yb;
  if (!x || !out || !out_scale || M <= 0 || K <= 0 || split <= 0 || lds < M) return YB_ERR_ARG;
  if (K % 128 != 0 || split % 128 != 0 || K % split != 0) return YB_ERR_SHAPE;
  if ((ldx % 8) || (split_stride % 8) || (ldo % 16) || (lds % 4) || (reinterpret_cast<uintptr_t>(x) & 0xF) ||
      (reinterpret_cast<uintptr_t>(out) & 0xF) || (reinterpret_cast<uintptr_t>(out_scale) & 0x3))
    return YB_ERR_ALIGNMENT;
  quant_rows_fp8_split_kernel<<<(M + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __nv_bfloat16*>(x), ldx, split, split_stride, static_cast<uint8_t*>(out), ldo,
      static_cast<float*>(out_scale), lds, M, K / 128);
  return check_launch("quant_rows_fp8_split");
}
