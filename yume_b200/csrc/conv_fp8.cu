// conv_fp8.cu — the FP8 (e4m3) path of the Wan2.2 VAE decode convs on sm_90a (H100): a block-scaled wgmma implicit-GEMM causal
// conv with per-group promotion, and the RMS_norm + SiLU (+ 2x upsample) pass that produces its quantised input.
// Numerics and constraints: include/yume_b200_fp8_vae.h. Structure follows gemm_fp8.cu (persistent, warp-specialised, TMA ring)
// with the A operand of the bf16 conv (gemm.cu): a 4-D TMA box of 128 output voxels per tap, out-of-bounds zero fill.
//   warp 0               producer: lane 0 issues the TMA loads of one (tap, 128-channel group) k-group — A box {128 ch, TW, TH,
//                        TT} e4m3, B tile 128 x 128 e4m3 (128B swizzle: one 128-byte swizzle row is exactly one scale group) —
//                        and all 32 lanes gather the 128 scales of the tap-shifted voxels (0 outside the input) into the stage;
//                        the stage's full barrier counts the 32 lane arrivals and the TMA bytes
//   warpgroups 1-2       consumers, rows [64 * (wg - 1), +64): per k-group 4 x wgmma m64n128k32 into a fresh accumulator, wait,
//                        then promotion acc_p += s_a[voxel + tap] * acc (fp32 FMA); epilogue straight from the fragment registers
// The scales go through the producer's lanes, not TMA: a TMA box of fp32 needs a 16-byte inner extent, and narrow boxes (TW < 4)
// do occur at the small levels.
#include "yb_host.h"
#include "../../include/yume_b200_fp8_vae.h"
#include "yb_ptx.cuh"

namespace yb {
namespace {

constexpr int CF8_BLOCK_M = 128;                             // output voxels per tile (TT x TH x TW)
constexpr int CF8_BLOCK_N = 128;                             // output channels per tile
constexpr int CF8_BLOCK_K = 128;                             // one scale group of one tap
constexpr int CF8_THREADS = 384;
constexpr int CF8_GROUP_N = 8;                               // rasterisation as gemm.cu
constexpr int CF8_TILE_BYTES = 128 * 128;
constexpr int CF8_STAGES = 6;
constexpr int CF8_SCALE_BYTES = CF8_BLOCK_M * 4;
constexpr int CF8_SMEM_BYTES = 1024 + CF8_STAGES * (2 * CF8_TILE_BYTES + CF8_SCALE_BYTES) + 256;

struct ConvFp8Params {
  const float* x_scale;   // [inT, groups, H, W]
  const float* w_scale;   // [Cout]
  const float* bias;      // [Cout] or null
  __nv_bfloat16* out;
  long long ldo;
  const __nv_bfloat16* res;
  long long res_ld;
  int inT, H, W, groups;  // input extents (history frames included) and Cp / 128
  int T;                  // output frames
  int taps;                // kt * 9: the spatial taps are always 3 x 3
  int off_t, off_h, off_w;
  int TW, TH, TT, tiles_w, tiles_h;
  int lg_tw, lg_twh;       // log2 TW, log2 (TW * TH)
  int num_m_tiles, num_n_tiles;
};

__device__ __forceinline__ void cf8_tile_coords(int tile, int num_m_tiles, int num_n_tiles, int& m_tile, int& n_tile) {
  const int per_group = CF8_GROUP_N * num_m_tiles;
  const int g = tile / per_group;
  const int r = tile - g * per_group;
  const int n_first = g * CF8_GROUP_N;
  const int n_in_group = min(CF8_GROUP_N, num_n_tiles - n_first);
  m_tile = r / n_in_group;
  n_tile = n_first + (r - m_tile * n_in_group);
}

// D (64 x 128, fp32) (+)= A (64 x 32 e4m3, smem K-major) * B (128 x 32 e4m3, smem K-major)
__device__ __forceinline__ void cf8_wgmma_e4m3_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// four floats -> four e4m3 bytes in memory order (x0 first)
__device__ __forceinline__ uint32_t cf8_cvt_e4m3x4(float x0, float x1, float x2, float x3) {
  uint32_t r;
  asm("{\n\t.reg .b16 lo, hi;\n\t"
      "cvt.rn.satfinite.e4m3x2.f32 lo, %2, %1;\n\t"
      "cvt.rn.satfinite.e4m3x2.f32 hi, %4, %3;\n\t"
      "mov.b32 %0, {lo, hi};\n\t}\n"
      : "=r"(r) : "f"(x0), "f"(x1), "f"(x2), "f"(x3));
  return r;
}

// (inv, scale) of a group with max |x| == amax: see include/yume_b200_fp8.h
__device__ __forceinline__ void cf8_group_scale(float amax, float& inv, float& scale) {
  inv = __fdiv_rn(448.0f, amax);
  scale = __fdiv_rn(amax, 448.0f);
  if (!(inv <= 3.402823466e38f)) { inv = 0.f; scale = 0.f; }
}

template <int EPI>
__global__ void __launch_bounds__(CF8_THREADS, 1)
conv3d_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const ConvFp8Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* sscale = reinterpret_cast<float*>(smem + CF8_STAGES * 2 * CF8_TILE_BYTES);   // [stage][128]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sscale + CF8_STAGES * CF8_BLOCK_M);
  uint64_t* empty_bar = full_bar + CF8_STAGES;

  const int warp = threadIdx.x >> 5;
  // m tile -> origin (t0, h0, w0) of its TT x TH x TW output box
  auto box_origin = [&](int mt, int& t0, int& h0, int& w0) {
    const int per_t = p.tiles_h * p.tiles_w;
    const int it = mt / per_t;
    const int rem = mt - it * per_t;
    const int ih = rem / p.tiles_w;
    t0 = it * p.TT;
    h0 = ih * p.TH;
    w0 = (rem - ih * p.tiles_w) * p.TW;
  };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < CF8_STAGES; ++i) {
      mbar_init(&full_bar[i], 32);   // the 32 producer lanes (lane 0's arrival also brings the TMA byte count)
      mbar_init(&empty_bar[i], 8);   // the 8 consumer warps
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<48>();   // 128 x 48 + 256 x 224 <= 384 x 168, the registers the launch holds
    if (warp == 0) {
      // ------------------------------- producer (whole warp) -------------------------------
      const int lane = threadIdx.x & 31;
      const int num_tiles = p.num_m_tiles * p.num_n_tiles, num_kb = p.taps * p.groups;
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_tile, n_tile, t0, h0, w0;
        cf8_tile_coords(tile, p.num_m_tiles, p.num_n_tiles, m_tile, n_tile);
        box_origin(m_tile, t0, h0, w0);
        // the scales of k-group kb are fetched one k-group ahead, so their latency hides behind the slot wait and the TMA issue.
        // Box row r = (tt * TH + th) * TW + tw (TW, TH powers of two); the tap-shifted input voxel of row lane + 32 i is recomputed
        // per fetch: the producer has 48 registers
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
          float* ss = sscale + stage * CF8_BLOCK_M;
#pragma unroll
          for (int i = 0; i < 4; ++i) ss[lane + 32 * i] = cur[i];
          if (lane == 0) {
            const int tap = kb / p.groups, g = kb - tap * p.groups;
            const int dt = tap / 9, dh = (tap / 3) % 3, dw = tap % 3;
            uint8_t* sa = smem + stage * 2 * CF8_TILE_BYTES;
            mbar_arrive_expect_tx(&full_bar[stage], 2 * CF8_TILE_BYTES);
            tma_load_4d(sa, &tmA, &full_bar[stage], g * CF8_BLOCK_K, w0 + dw - p.off_w, h0 + dh - p.off_h, t0 + dt - p.off_t);
            tma_load_2d(sa + CF8_TILE_BYTES, &tmB, &full_bar[stage], kb * CF8_BLOCK_K, n_tile * CF8_BLOCK_N);
          } else {
            mbar_arrive(&full_bar[stage]);
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) cur[i] = nxt[i];
          if (++stage == CF8_STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ------------------------------- consumers: MMA + promotion + epilogue -------------------------------
    setmaxnreg_inc<224>();
    const int lane = threadIdx.x & 31;
    const int num_tiles = p.num_m_tiles * p.num_n_tiles, num_kb = p.taps * p.groups;
    const int wg = (warp >> 2) - 1;
    const int q4 = lane >> 2, c2 = 2 * (lane & 3);   // fragment: rows q4 / q4 + 8 of the warp's 16, columns 8g + c2, +1
    const int r_lo = wg * 64 + (warp & 3) * 16 + q4;  // tile row of this thread's first fragment row
    int stage = 0;
    uint32_t phase = 0;
    float acc[64], accp[64];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int m_tile, n_tile;
      cf8_tile_coords(tile, p.num_m_tiles, p.num_n_tiles, m_tile, n_tile);
#pragma unroll
      for (int i = 0; i < 64; ++i) accp[i] = 0.f;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * 2 * CF8_TILE_BYTES);
        const uint64_t ad = make_smem_desc_sw128(sa + wg * 64 * 128, 16, 1024);
        const uint64_t bd = make_smem_desc_sw128(sa + CF8_TILE_BYTES, 16, 1024);
        fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < CF8_BLOCK_K / 32; ++k) cf8_wgmma_e4m3_n128(acc, ad + 2 * k, bd + 2 * k, k == 0 ? 0u : 1u);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(acc);
        const float s_lo = sscale[stage * CF8_BLOCK_M + r_lo];
        const float s_hi = sscale[stage * CF8_BLOCK_M + r_lo + 8];
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == CF8_STAGES) {
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

      // ---- epilogue: v = accp * s_w[n] + bias[n] (+ res), bf16, straight from the fragment; rows outside the output are skipped
      int t0, h0, w0;
      {
        const int per_t = p.tiles_h * p.tiles_w;
        const int it = m_tile / per_t;
        const int rem = m_tile - it * per_t;
        const int ih = rem / p.tiles_w;
        t0 = it * p.TT;
        h0 = ih * p.TH;
        w0 = (rem - ih * p.tiles_w) * p.TW;
      }
      long long orow[2];
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int r = r_lo + 8 * half;
        const int t = t0 + (r >> p.lg_twh), h = h0 + ((r >> p.lg_tw) & (p.TH - 1)), w = w0 + (r & (p.TW - 1));
        orow[half] = (t < p.T && h < p.H && w < p.W) ? (static_cast<long long>(t) * p.H + h) * p.W + w : -1;
      }
      const int n0 = n_tile * CF8_BLOCK_N;
#pragma unroll
      for (int g = 0; g < 16; ++g) {
        const int col = n0 + 8 * g + c2;
        const float2 sw = __ldg(reinterpret_cast<const float2*>(p.w_scale + col));
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
    }
  }
}

// ------------------------------------------------------------------------------------------------
// RMS_norm (* gamma) -> SiLU -> nearest 2x upsample -> bf16 rounding -> 1x128 e4m3 quantisation per voxel.
// Lane layout and fp32 arithmetic are those of rms_act_kernel<NCH, G> (vae_elementwise.cu) for the same C / Cp, so the bf16 values
// are the ones yb_vae_rms_act stores. Chunk c (8 channels) of a voxel sits on lane gl = c % G, so the 16 chunks of one 128-channel
// group are 16 adjacent lanes (G is 16 or 32 here): the group max is a 4-step shuffle over them.
// ------------------------------------------------------------------------------------------------
template <int NCH, int G>
__global__ void __launch_bounds__(256, 2)
rms_act_fp8_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, uint8_t* __restrict__ out, float* __restrict__ out_scale,
                   const float* __restrict__ gamma, int T, int Hs, int Ws, int C, int Cp, int f, int silu) {
  static_assert(G == 16 || G == 32, "a 128-channel group spans 16 lanes");
  constexpr int U = 4 / NCH;
  constexpr int SUB = 32 / G;
  constexpr int VPI = U * SUB;
  const int H = Hs * f, W = Ws * f;
  const int HW = H * W;
  const int nvox = T * HW;
  const int lane = threadIdx.x & 31;
  const int gl = lane % G, sub = lane / G;
  const int cch = C >> 3, pch = Cp >> 3;
  const int groups = Cp >> 7;
  const float sqrt_c = sqrtf(static_cast<float>(C));
  const int stride = gridDim.x * 8 * VPI;
  for (int v0 = (blockIdx.x * 8 + (threadIdx.x >> 5)) * VPI; v0 < nvox; v0 += stride) {
    uint4 raw[U][NCH];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int v = v0 + u * SUB + sub;
      int src = v;
      if (f != 1) {
        const int w = v % W, r = v / W;
        const int h = r % H, t = r / H;
        src = (t * Hs + h / f) * Ws + w / f;
      }
      const __nv_bfloat16* xs = x + static_cast<long long>(src) * ldx;
#pragma unroll
      for (int j = 0; j < NCH; ++j) {
        const int c = gl + G * j;
        raw[u][j] = (v < nvox && c < cch) ? *reinterpret_cast<const uint4*>(xs + c * 8) : make_uint4(0u, 0u, 0u, 0u);
      }
    }
    float scl[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float ss = 0.f;
#pragma unroll
      for (int j = 0; j < NCH; ++j) {
        const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&raw[u][j]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 a = __bfloat1622float2(hh[k]);
          ss += a.x * a.x + a.y * a.y;
        }
      }
      scl[u] = ss;
    }
    if (gamma) {
#pragma unroll
      for (int o = G / 2; o > 0; o >>= 1) {
#pragma unroll
        for (int u = 0; u < U; ++u) scl[u] += __shfl_xor_sync(0xffffffffu, scl[u], o);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int v = v0 + u * SUB + sub;   // every lane takes part in the shuffles below; only the stores check v
      const float sc = gamma ? sqrt_c / fmaxf(sqrtf(scl[u]), 1e-12f) : 1.f;
#pragma unroll
      for (int j = 0; j < NCH; ++j) {
        const int c = gl + G * j;
        float y[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (c < cch) {
          const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&raw[u][j]);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float2 a = __bfloat1622float2(hh[k]);
            y[2 * k] = a.x;
            y[2 * k + 1] = a.y;
          }
          if (gamma) {
            const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c * 8));
            const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + c * 8 + 4));
            const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
            for (int k = 0; k < 8; ++k) y[k] = y[k] * sc * gg[k];
          }
          if (silu) {
#pragma unroll
            for (int k = 0; k < 8; ++k) y[k] = y[k] / (1.f + __expf(-y[k]));
          }
#pragma unroll
          for (int k = 0; k < 8; ++k) y[k] = __bfloat162float(__float2bfloat16_rn(y[k]));   // the value yb_vae_rms_act stores
        }
        float amax = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) amax = fmaxf(amax, fabsf(y[k]));
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        if (v >= nvox || c >= pch) continue;
        float inv, scale;
        cf8_group_scale(amax, inv, scale);
        *reinterpret_cast<uint2*>(out + static_cast<long long>(v) * Cp + c * 8) =
            make_uint2(cf8_cvt_e4m3x4(y[0] * inv, y[1] * inv, y[2] * inv, y[3] * inv),
                       cf8_cvt_e4m3x4(y[4] * inv, y[5] * inv, y[6] * inv, y[7] * inv));
        if ((c & 15) == 0) {
          const int t = v / HW;
          out_scale[(static_cast<long long>(t) * groups + (c >> 4)) * HW + (v - t * HW)] = scale;
        }
      }
    }
  }
}

// 4-D e4m3 tensor map over a dense channels-last volume [T, H, W, C] (C bytes per voxel), box {128 channels, bw, bh, bt}, 128-byte
// swizzle, out-of-bounds voxels read as zeros
int make_tmap_e4m3_4d(CUtensorMap* tm, const void* base, uint64_t T, uint64_t H, uint64_t W, uint64_t C, uint32_t bt, uint32_t bh,
                      uint32_t bw) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return YB_ERR_NO_DRIVER;
  if ((reinterpret_cast<uintptr_t>(base) & 0xF) || (C & 0xF)) return YB_ERR_ALIGNMENT;
  cuuint64_t gdim[4] = {C, W, H, T};
  cuuint64_t gstride[3] = {C, W * C, H * W * C};
  cuuint32_t box[4] = {CF8_BLOCK_K, bw, bh, bt};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  if (bw > 256 || bh > 256 || bt > 256) return YB_ERR_SHAPE;
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? YB_OK : YB_ERR_TENSORMAP;
}

// e4m3 weight [Cout, K] (row stride K bytes), box 128 x 128, 128-byte swizzle
int make_tmap_e4m3_w(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t K) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return YB_ERR_NO_DRIVER;
  if ((reinterpret_cast<uintptr_t>(base) & 0xF) || (K & 0xF)) return YB_ERR_ALIGNMENT;
  cuuint64_t gdim[2] = {K, rows};
  cuuint64_t gstride[1] = {K};
  cuuint32_t box[2] = {CF8_BLOCK_K, CF8_BLOCK_N};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? YB_OK : YB_ERR_TENSORMAP;
}

template <int EPI>
int launch_conv3d_fp8(const CUtensorMap& tmA, const CUtensorMap& tmB, const ConvFp8Params& p, cudaStream_t stream) {
  static bool attr_set[kMaxDevices] = {};
  if (int rc = ensure_dynamic_smem(conv3d_fp8_kernel<EPI>, CF8_SMEM_BYTES, attr_set, "conv3d_fp8")) return rc;
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  const int grid = tiles < sm_count() ? tiles : sm_count();
  conv3d_fp8_kernel<EPI><<<grid, CF8_THREADS, CF8_SMEM_BYTES, stream>>>(tmA, tmB, p);
  return check_launch("conv3d_fp8");
}

}  // namespace
}  // namespace yb

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
  ConvFp8Params p;
  p.TW = plan[0];
  p.TH = plan[1];
  p.TT = plan[2];
  p.x_scale = static_cast<const float*>(a->x_scale);
  p.w_scale = static_cast<const float*>(a->w_scale);
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
  p.num_n_tiles = a->Cout / CF8_BLOCK_N;
  CUtensorMap tmA, tmB;
  int rc = make_tmap_e4m3_4d(&tmA, a->x, inT, a->H, a->W, a->Cp, p.TT, p.TH, p.TW);
  if (rc) return rc;
  rc = make_tmap_e4m3_w(&tmB, a->w, a->Cout, static_cast<uint64_t>(p.taps) * a->Cp);
  if (rc) return rc;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (a->epilogue == YB_EPI_RES_BF16) return launch_conv3d_fp8<YB_EPI_RES_BF16>(tmA, tmB, p, stream);
  return launch_conv3d_fp8<YB_EPI_BF16>(tmA, tmB, p, stream);
}

extern "C" int yb_vae_rms_act_fp8(const void* x, long long ldx, void* out, void* out_scale, const void* gamma, int T, int Hs, int Ws,
                                  int C, int Cp, int up, int silu, void* stream_) {
  using namespace yb;
  if (!x || !out || !out_scale || T <= 0 || Hs <= 0 || Ws <= 0 || C <= 0) return YB_ERR_ARG;
  if (C % 8 != 0 || C > 1024 || Cp % 128 != 0 || Cp != (C + 127) / 128 * 128 || (up != 1 && up != 2)) return YB_ERR_SHAPE;
  if ((ldx % 8) || (reinterpret_cast<uintptr_t>(x) & 0xF) || (reinterpret_cast<uintptr_t>(out) & 0xF) ||
      (reinterpret_cast<uintptr_t>(out_scale) & 0x3))
    return YB_ERR_ALIGNMENT;
  if (gamma && (reinterpret_cast<uintptr_t>(gamma) & 0xF)) return YB_ERR_ALIGNMENT;
  const long long nvox = static_cast<long long>(T) * Hs * up * Ws * up;
  if (nvox > 0x7fffffffLL - (1LL << 24)) return YB_ERR_SHAPE;
  // the (NCH, G) instance yb_vae_rms_act takes for this C / Cp (Cp >= 128 here, so G is 16 or 32)
  const int nch = C <= 256 ? 1 : (C <= 512 ? 2 : 4);
  const int g = nch > 1 ? 32 : (Cp <= 128 ? 16 : 32);
  const int per_block = 8 * (4 / nch) * (32 / g);
  long long blocks = (nvox + per_block - 1) / per_block;
  if (blocks > static_cast<long long>(sm_count()) * 32) blocks = static_cast<long long>(sm_count()) * 32;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
#define YB_RMS8_LAUNCH(NCH, G)                                                                                          \
  rms_act_fp8_kernel<NCH, G><<<static_cast<int>(blocks), 256, 0, st>>>(                                                 \
      static_cast<const __nv_bfloat16*>(x), ldx, static_cast<uint8_t*>(out), static_cast<float*>(out_scale),            \
      static_cast<const float*>(gamma), T, Hs, Ws, C, Cp, up, silu)
  if (nch == 4) YB_RMS8_LAUNCH(4, 32);
  else if (nch == 2) YB_RMS8_LAUNCH(2, 32);
  else if (g == 32) YB_RMS8_LAUNCH(1, 32);
  else YB_RMS8_LAUNCH(1, 16);
#undef YB_RMS8_LAUNCH
  return check_launch("vae_rms_act_fp8");
}
