// attention_fp8.cu — the e4m3 self-attention of precision="fp8_attn" on sm_90a (H100): the V quantiser that writes V
// transposed (the K-major B operand e4m3 wgmma requires) with per-(head, 128-key tile) scales, and the attention kernel.
// Numerics and constraints: include/yume_b200_fp8_attn.h. Structure follows attention.cu (same work units, the same TMA
// producer and two consumer warpgroups, the same intra-warpgroup overlap of S_{j+1} with P_j V_j, the same tail split and
// combine):
//   warpgroup 0     TMA producer (one thread): Q8 tile (16 KB) + its 128 q scales, then K8_j (16 KB) + its 128 k scales and
//                   Vt8_j (16 KB) through an smem ring
//   warpgroups 1-2  query rows [64*(wg-1), +64) of the current tile:
//                   S = Q8 K8_j^T           4 x wgmma m64n128k32 e4m3 (both operands in smem) into a fresh accumulator
//                   s = S * s_k[key]        per column, then masking and the online softmax with the row factor
//                                           s_q * scale * log2(e) folded into the exp2 FFMA
//                   P8 = e4m3(256 p)        packed inside the thread: Vt8 stores the keys of every 32-key block in the order pi
//                                           (header), so the accumulator fragment already holds the keys of the A fragment
//                   O_tile = P8 Vt8_j       4 x wgmma m64n128k32 e4m3, A from registers, into a fresh accumulator
//                   O = O alpha + O_tile s_v[j]   promotion in fp32 (the e4m3 tensor-core accumulator keeps 13 mantissa bits)
//
// Consumer schedule per query tile of nkv KV tiles (attention.cu's, with the promotion after the P V wait):
//   prologue   issue S_0, wait, s *= s_k, release K_0, softmax(S_0) in place, pack P_0
//   step j     issue S_{j+1} (not on the last step); issue O_tile = P_j V_j;
//              wait<1> (S_{j+1} retired) -> s *= s_k, release K_{j+1}, softmax(S_{j+1}) in place while P_j V_j runs;
//              wait<0> -> release V_j, pack P_{j+1}, O = (O + O_tile s_v[j]) alpha_{j+1}, the multiply skipped when alpha is
//              1 for every row of the warp (an identity; the common case once the running maxima settle)
// Live: O, S and O_tile (64 registers each) and P8 (16); the consumers take 240 registers (setmaxnreg), the producer 24.
// The k scales live in K_{j+1}'s ring slot, so they are applied before the slot is released. The exponentials are computed as
// 2^(x - m + 8) = 256 p directly; l sums them unrounded, so l and O both carry the factor 256, which cancels in O / l and is
// taken out (exactly) of the KV-split partials, which are written in true units.
//
// Barriers: attention.cu's protocol with its counts (q_full / q_empty, kv_full[s] / kv_empty[s], one global ring sequence it:
// K_j of query tile X at it, V_j at it + 1). q_full and K-slot kv_full expect the tile plus its 512 B of scales.
#include "yb_host.h"
#include "../../include/yume_b200_fp8.h"
#include "../../include/yume_b200_fp8_attn.h"
#include "../../include/yume_b200_fp8_sp.h"
#include "yb_ptx.cuh"

namespace yb {

constexpr int A8_THREADS = 384;
constexpr int A8_TILE_BYTES = 128 * 128;   // one 128 x 128 e4m3 tile = one 128B-swizzled slab
constexpr int A8_NS = 8;                   // KV ring slots (K and Vt tiles alternate)
constexpr int A8_Q_OFF = 0;
constexpr int A8_KV_OFF = A8_TILE_BYTES;
constexpr int A8_QS_OFF = A8_KV_OFF + A8_NS * A8_TILE_BYTES;   // f32 [2][128] q scales of query tiles 0 and 1
constexpr int A8_KS_OFF = A8_QS_OFF + 1024;                     // f32 [A8_NS][128] k scales (K slots only)
constexpr int A8_BAR_OFF = A8_KS_OFF + A8_NS * 512;
constexpr int A8_SINK_OFF = A8_BAR_OFF + 256;
static_assert((2 + 2 * A8_NS) * 8 <= 256, "mbarriers below the sink word");
constexpr int A8_SMEM_BYTES = A8_BAR_OFF + 512 + 1024;
static_assert(A8_SMEM_BYTES <= 227 * 1024, "shared memory budget");

struct Att8Params {
  __nv_bfloat16* out;
  long long ldo;
  int Lq, Lk, heads, nkv;
  const float* v_scale;   // [heads, nkv]
  float scale_log2;       // softmax scale * log2(e)
  int nq, full_units, ns; // work decomposition as attention.cu's AttParams
  float* ws_o;            // [tail CTAs, 256, 128] O in true units
  float* ws_ml;           // [tail CTAs, 256, 2]   (row max in the log2 domain, row sum of p)
};

// D (64 x 128, fp32) (+)= A (64 x 32 e4m3, registers) * B (128 x 32 e4m3, smem K-major). A fragment of the thread (lane l of
// warp w, t = l % 4): a[0] row 16w + l/4, k 4t .. 4t+3 (byte 0 first); a[1] the row 8 further down; a[2], a[3] the same at
// k 16 + 4t .. 16 + 4t + 3.
__device__ __forceinline__ void wgmma_rs_e4m3(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}

// tile row of the thread's fragment row a (row b = + 8) for the consumer warpgroups, re-derived from %tid.x at each use: a
// value held across the KV loop is what ptxas spills first in this kernel
__device__ __forceinline__ int a8_row_a() {
  uint32_t t;
  asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
  return static_cast<int>((t >> 7) - 1) * 64 + static_cast<int>((t >> 5) & 3) * 16 + static_cast<int>((t & 31) >> 2);
}

// Ulysses (yb_attention_fp8_sp): output row g belongs to rank g / Lp and is stored into row rank * Lp + g % Lp of that rank's
// [P(src), Lp, heads_local * 128] receive buffer over NVLink, as attention.cu's AttParams.out_peers
struct Att8Peers {
  __nv_bfloat16* out[8];
  int world, rank, Lp;
};

// the kernel body; SP selects the epilogue's store address (attention_fp8_kernel / attention_fp8_sp_kernel), nothing else
template <bool SP>
__device__ __forceinline__ void attention_fp8_body(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                                                   const CUtensorMap& tmSQ, const CUtensorMap& tmSK, const Att8Params& p,
                                                   const Att8Peers* sp) {
  constexpr int NS = A8_NS;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + A8_BAR_OFF);
  uint64_t* q_empty = q_full + 1;
  uint64_t* kv_full = q_empty + 1;
  uint64_t* kv_empty = kv_full + NS;
  const float* qsc = reinterpret_cast<const float*>(smem + A8_QS_OFF);
  const float* ksc = reinterpret_cast<const float*>(smem + A8_KS_OFF);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  int unit = blockIdx.x, kv_begin = 0, nkv = p.nkv;
  if (static_cast<int>(blockIdx.x) >= p.full_units) {   // KV segment of a tail unit (attention.cu's decomposition)
    const int r = blockIdx.x - p.full_units;
    unit = p.full_units + r / p.ns;
    const int per = (((p.nkv + p.ns - 1) / p.ns) + 1) & ~1;
    kv_begin = (r % p.ns) * per;
    nkv = min(per, p.nkv - kv_begin);
  }
  const int head = unit / p.nq;
  const int q0 = (unit - head * p.nq) * 256;
  const int nx = q0 + 128 < p.Lq ? 2 : 1;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmSQ);
    tma_prefetch_desc(&tmSK);
    mbar_init(q_full, 1);
    mbar_init(q_empty, 8);
    for (int i = 0; i < NS; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<24>();
    if (warp == 0 && lane == 0) {
      // ------------------------------- TMA producer -------------------------------
      int it = 0;
      for (int X = 0; X < nx; ++X) {
        if (X == 1) mbar_wait(q_empty, 0);
        mbar_arrive_expect_tx(q_full, A8_TILE_BYTES + 512);
        tma_load_2d(smem + A8_Q_OFF, &tmQ, q_full, head * 128, q0 + X * 128);
        tma_load_2d(smem + A8_QS_OFF + X * 512, &tmSQ, q_full, q0 + X * 128, head);
        for (int jj = 0; jj < 2 * nkv; ++jj, ++it) {
          const int slot = it % NS;
          const int j = kv_begin + (jj >> 1);
          mbar_wait(&kv_empty[slot], ((it / NS) & 1) ^ 1);
          uint8_t* dst = smem + A8_KV_OFF + slot * A8_TILE_BYTES;
          if (jj & 1) {
            mbar_arrive_expect_tx(&kv_full[slot], A8_TILE_BYTES);
            tma_load_2d(dst, &tmV, &kv_full[slot], j * 128, head * 128);
          } else {
            mbar_arrive_expect_tx(&kv_full[slot], A8_TILE_BYTES + 512);
            tma_load_2d(dst, &tmK, &kv_full[slot], head * 128, j * 128);
            tma_load_2d(smem + A8_KS_OFF + slot * 512, &tmSK, &kv_full[slot], j * 128, p.heads + head);
          }
        }
      }
    }
  } else {
    // ------------------------------- S, softmax, P V, promotion, epilogue -------------------------------
    setmaxnreg_inc<240>();
    const int wg = (warp >> 2) - 1;
    const int c2 = 2 * (lane & 3);   // fragment columns 8g + c2, +1
    const uint32_t sQ = smem_u32(smem + A8_Q_OFF) + wg * 64 * 128;
    auto issue_s = [&](float (&s)[64], int itk) {
      const int slot_k = itk % NS;
      att_wait(&kv_full[slot_k], (itk / NS) & 1);
      const uint32_t sK = smem_u32(smem + A8_KV_OFF + slot_k * A8_TILE_BYTES);
      const uint64_t qd = make_smem_desc_sw128(sQ, 16, 1024), kd = make_smem_desc_sw128(sK, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_ss_e4m3(s, qd + 2 * kk, kd + 2 * kk, kk != 0);   // 32 B per k-step
      wgmma_commit();
    };
    int it = 0;
    for (int X = 0; X < nx; ++X) {
      att_wait(q_full, X);
      float o[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) o[i] = 0.f;
      float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // running max (log2 domain), sum of 256 p
      float al0, al1;
      float s[64];         // S of one KV tile, overwritten in place by 256 p
      float ot[64];        // O_tile = P8 Vt8_j
      uint32_t pa[4][4];   // P8 as the A fragments of the 4 k-steps of P V
      // S of the K tile in `slot` times the k scale of each column; columns past Lk count as -inf
      auto scale_k = [&](int slot, int j) {
        const float* sk = ksc + slot * 128 + c2;
#pragma unroll
        for (int g = 0; g < 16; ++g) {
          const float2 kv = *reinterpret_cast<const float2*>(sk + 8 * g);
          s[4 * g] *= kv.x;
          s[4 * g + 1] *= kv.y;
          s[4 * g + 2] *= kv.x;
          s[4 * g + 3] *= kv.y;
        }
        const int kv_rem = p.Lk - (kv_begin + j) * 128;
        if (kv_rem < 128) {
#pragma unroll
          for (int i = 0; i < 64; ++i)
            if (8 * (i >> 2) + c2 + (i & 1) >= kv_rem) s[i] = -INFINITY;
        }
      };
      auto softmax = [&]() {
        // row factors s_q * scale * log2(e), read from shared memory each time rather than held in registers (each query tile
        // has its own q scales, so they outlive the reload of Q); a zero q scale (an all-zero row) keeps a tiny positive
        // factor so that masked columns stay -inf instead of becoming 0 * -inf
        const float* qs = qsc + X * 128 + a8_row_a();
        const float rq0 = fmaxf(qs[0] * p.scale_log2, 1e-30f);
        const float rq1 = fmaxf(qs[8] * p.scale_log2, 1e-30f);
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int g = 0; g < 16; ++g) {
          mx0 = fmaxf(mx0, fmaxf(s[4 * g], s[4 * g + 1]));
          mx1 = fmaxf(mx1, fmaxf(s[4 * g + 2], s[4 * g + 3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float mn0 = fmaxf(m0, mx0 * rq0), mn1 = fmaxf(m1, mx1 * rq1);
        al0 = fast_exp2(m0 - mn0);
        al1 = fast_exp2(m1 - mn1);
        m0 = mn0;
        m1 = mn1;
        l0 *= al0;
        l1 *= al1;
        const float b0 = 8.0f - m0, b1 = 8.0f - m1;   // 2^(x - m + 8) = 256 p
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
          float* e = s + 8 * kk;
#pragma unroll
          for (int i = 0; i < 8; ++i) e[i] = fast_exp2(fmaf(e[i], (i & 2) ? rq1 : rq0, (i & 2) ? b1 : b0));
          l0 += (e[0] + e[1]) + (e[4] + e[5]);
          l1 += (e[2] + e[3]) + (e[6] + e[7]);
        }
      };
      // 256 p -> e4m3 A fragments. k-step kk covers stored positions [32kk, 32kk + 32), which hold keys 32kk + pi(f): the
      // thread's accumulator columns 32kk + {2t, 2t+1, 8+2t, 9+2t} feed positions 4t .. 4t+3, columns 32kk + 16 + the same feed
      // positions 16 + 4t .. 16 + 4t + 3
      auto pack_p = [&]() {
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const float* e = s + 16 * kk;
          pa[kk][0] = cvt_e4m3x4(e[0], e[1], e[4], e[5]);       // row a
          pa[kk][1] = cvt_e4m3x4(e[2], e[3], e[6], e[7]);       // row b
          pa[kk][2] = cvt_e4m3x4(e[8], e[9], e[12], e[13]);     // row a, +16
          pa[kk][3] = cvt_e4m3x4(e[10], e[11], e[14], e[15]);   // row b, +16
        }
      };

      issue_s(s, it);
      wgmma_wait<0>();
      fence_regs(s);
      scale_k(it % NS, 0);
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&kv_empty[it % NS]);
        if (nkv == 1) mbar_arrive(q_empty);
      }
      softmax();
      pack_p();
      auto kv_step = [&](int j, const bool next) {
        const int slot_v = (it + 1) % NS, slot_kn = (it + 2) % NS;
        if (next) issue_s(s, it + 2);
        att_wait(&kv_full[slot_v], ((it + 1) / NS) & 1);
        const uint64_t vd = make_smem_desc_sw128(smem_u32(smem + A8_KV_OFF + slot_v * A8_TILE_BYTES), 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs_e4m3(ot, pa[kk], vd + 2 * kk, kk != 0);
        wgmma_commit();
        if (next) {
          wgmma_wait<1>();
          fence_regs(s);
          scale_k(slot_kn, j + 1);
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(&kv_empty[slot_kn]);
            if (j + 2 == nkv) mbar_arrive(q_empty);
          }
          softmax();
          // keeps ptxas from hoisting the wait below above the softmax (see attention.cu)
          if (l0 + l1 < 0.f) *reinterpret_cast<volatile float*>(smem + A8_SINK_OFF) = l0;
        }
        wgmma_wait<0>();
        fence_regs(ot);
        __syncwarp();
        if (lane == 0) mbar_arrive(&kv_empty[slot_v]);
        if (next) pack_p();   // pa was P_j V_j's operand until now
        // promotion, with O already scaled by alpha_j: O = O + O_tile s_v[j], then alpha_{j+1} of the next tile. Once the
        // running maxima settle, alpha is 1 for every row of the warp and the multiply (an identity then) is skipped
        const float sv = __ldg(p.v_scale + static_cast<long long>(head) * p.nkv + kv_begin + j);
#pragma unroll
        for (int i = 0; i < 64; ++i) o[i] = fmaf(ot[i], sv, o[i]);
        if (next && __any_sync(0xffffffffu, al0 != 1.f || al1 != 1.f)) {
#pragma unroll
          for (int g = 0; g < 16; ++g) {
            o[4 * g] *= al0;
            o[4 * g + 1] *= al0;
            o[4 * g + 2] *= al1;
            o[4 * g + 3] *= al1;
          }
        }
        it += 2;
      };
      for (int j = 0; j + 1 < nkv; ++j) kv_step(j, true);
      kv_step(nkv - 1, false);
      l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
      l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 2);

      // epilogue: O / l -> bf16 -> global [Lq, heads*128], or (O, m, l) / 256 -> the KV-segment workspace
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row_t = X * 128 + a8_row_a() + 8 * h;
        const float m = h ? m1 : m0, l = h ? l1 : l0;
        if (static_cast<int>(blockIdx.x) >= p.full_units) {
          const long long prow = static_cast<long long>(blockIdx.x - p.full_units) * 256 + row_t;
          float* wo = p.ws_o + prow * 128;
#pragma unroll
          for (int g = 0; g < 16; ++g)
            *reinterpret_cast<float2*>(wo + 8 * g + c2) =
                make_float2(o[4 * g + 2 * h] * 0.00390625f, o[4 * g + 2 * h + 1] * 0.00390625f);
          if ((lane & 3) == 0) *reinterpret_cast<float2*>(p.ws_ml + prow * 2) = make_float2(m, l * 0.00390625f);
          continue;
        }
        const int q_row = q0 + row_t;
        if (q_row >= p.Lq) continue;
        // the column offset is formed here from %laneid: hoisted above the KV loop, ptxas would spill it
        uint32_t ln;
        asm volatile("mov.u32 %0, %%laneid;" : "=r"(ln));
        const int col0 = head * 128 + 2 * static_cast<int>(ln & 3);
        __nv_bfloat16* orow;
        if constexpr (SP) {
          const int owner = q_row / sp->Lp;   // < world: Lq == world * Lp
          orow = sp->out[owner] + (static_cast<long long>(sp->rank) * sp->Lp + (q_row - owner * sp->Lp)) * p.ldo + col0;
        } else {
          orow = p.out + static_cast<long long>(q_row) * p.ldo + col0;
        }
        const float inv = 1.0f / l;
#pragma unroll
        for (int g = 0; g < 16; ++g)
          *reinterpret_cast<uint32_t*>(orow + 8 * g) = pack_bf16x2(o[4 * g + 2 * h] * inv, o[4 * g + 2 * h + 1] * inv);
      }
    }
  }
}

__global__ void __launch_bounds__(A8_THREADS, 1)
attention_fp8_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmSQ,
                     const __grid_constant__ CUtensorMap tmSK, const Att8Params p) {
  attention_fp8_body<false>(tmQ, tmK, tmV, tmSQ, tmSK, p, nullptr);
}

__global__ void __launch_bounds__(A8_THREADS, 1)
attention_fp8_sp_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmSQ,
                        const __grid_constant__ CUtensorMap tmSK, const Att8Params p, const __grid_constant__ Att8Peers sp) {
  attention_fp8_body<true>(tmQ, tmK, tmV, tmSQ, tmSK, p, &sp);
}

// ------------------------------------------------------------------------------------------------
// V -> Vt8 + per-(head, 128-key tile) scales. One CTA per (key tile, head): the 128 x 128 bf16 block is staged in shared memory
// (keys >= Lk as zeros), its amax taken over all 16384 values (NaN ignored), then every thread writes 64 consecutive stored
// positions of one output row d.
// ------------------------------------------------------------------------------------------------
constexpr int VT_PITCH = 136;   // bf16 per staged row: 272 B keeps 16-byte stores aligned and shifts rows by 4 banks

__host__ __device__ constexpr int vt_pi(int f) { return 16 * (f >> 4) + 2 * ((f & 15) >> 2) + 8 * ((f & 3) >> 1) + (f & 1); }

__global__ void __launch_bounds__(256)
quant_vt_fp8_kernel(const __nv_bfloat16* __restrict__ v, long long ldv, uint8_t* __restrict__ vt8, float* __restrict__ v_scale,
                    int Lk, int Lkp) {
  __shared__ __align__(16) __nv_bfloat16 tile[128 * VT_PITCH];
  __shared__ float wmax[8];
  const int j = blockIdx.x, head = blockIdx.y;
  const int tid = threadIdx.x;
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {   // 2048 chunks of 8 bf16: row = chunk / 16, 8 columns at (chunk % 16) * 8
    const int c = tid + 256 * i;
    const int r = c >> 4, col = (c & 15) * 8;
    const int key = j * 128 + r;
    uint4 raw = make_uint4(0u, 0u, 0u, 0u);
    if (key < Lk) raw = __ldg(reinterpret_cast<const uint4*>(v + static_cast<long long>(key) * ldv + head * 128 + col));
    *reinterpret_cast<uint4*>(tile + r * VT_PITCH + col) = raw;
    const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __bfloat1622float2(h2[e]);
      amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));   // fmaxf drops a NaN operand
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if ((tid & 31) == 0) wmax[tid >> 5] = amax;
  __syncthreads();
  amax = wmax[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) amax = fmaxf(amax, wmax[w]);
  float inv, sc;
  group_scale(amax, inv, sc);
  if (tid == 0) v_scale[static_cast<long long>(head) * (Lkp / 128) + j] = sc;
  const int d = tid & 127, f0 = (tid >> 7) * 64;
  uint8_t* orow = vt8 + (static_cast<long long>(head) * 128 + d) * Lkp + j * 128 + f0;
#pragma unroll
  for (int c = 0; c < 4; ++c) {   // 16 stored positions per 16-byte store
    uint32_t w[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float x[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int f = f0 + 16 * c + 4 * q + e;
        const int key = 32 * (f >> 5) + vt_pi(f & 31);
        x[e] = __bfloat162float(tile[key * VT_PITCH + d]) * inv;
      }
      w[q] = cvt_e4m3x4(x[0], x[1], x[2], x[3]);
    }
    *reinterpret_cast<uint4*>(orow + 16 * c) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

}  // namespace yb

extern "C" int yb_quant_vt_fp8(const void* v, long long ldv, void* vt8, void* v_scale, int Lk, int heads, void* stream_) {
  using namespace yb;
  if (!v || !vt8 || !v_scale || Lk <= 0 || heads <= 0) return YB_ERR_ARG;
  if ((ldv % 8) || (reinterpret_cast<uintptr_t>(v) & 0xF) || (reinterpret_cast<uintptr_t>(vt8) & 0xF) ||
      (reinterpret_cast<uintptr_t>(v_scale) & 0x3))
    return YB_ERR_ALIGNMENT;
  const int Lkp = (Lk + 127) / 128 * 128;
  quant_vt_fp8_kernel<<<dim3(Lkp / 128, heads), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __nv_bfloat16*>(v), ldv, static_cast<uint8_t*>(vt8), static_cast<float*>(v_scale), Lk, Lkp);
  return check_launch("quant_vt_fp8");
}

namespace yb {

// yb_attention_fp8 and yb_attention_fp8_sp: sp == nullptr stores rows into `out`, otherwise into the owners' receive buffers
static int launch_attention_fp8(const void* q8, long long ldq, const void* k8, long long ldk, const void* qk_scale, long long lds,
                                const void* vt8, const void* v_scale, void* out, long long ldo, int Lq, int Lk, int heads,
                                float scale, int flags, void* ws, long long ws_bytes, const Att8Peers* sp, void* stream_) {
  if (!q8 || !k8 || !qk_scale || !vt8 || !v_scale || !out) return YB_ERR_ARG;
  if (Lq <= 0 || Lk <= 0 || heads <= 0 || lds < Lq || lds < Lk) return YB_ERR_ARG;
  if (flags & ~(7 << YB_ATT_SPLIT_SHIFT)) return YB_ERR_ARG;   // no accumulate, P-in-smem or emulation forms
  if (((flags >> YB_ATT_SPLIT_SHIFT) & 7) > 4) return YB_ERR_ARG;
  if ((ldo % 8) || (reinterpret_cast<uintptr_t>(out) & 0xF) || (reinterpret_cast<uintptr_t>(v_scale) & 0x3))
    return YB_ERR_ALIGNMENT;
  const int nkv = (Lk + 127) / 128;
  const uint64_t cols = static_cast<uint64_t>(heads) * 128;
  CUtensorMap tmQ, tmK, tmV, tmSQ, tmSK;
  int rc = make_tmap_e4m3_2d(&tmQ, q8, Lq, cols, ldq);
  if (rc) return rc;
  rc = make_tmap_e4m3_2d(&tmK, k8, Lk, cols, ldk);
  if (rc) return rc;
  rc = make_tmap_e4m3_2d(&tmV, vt8, cols, static_cast<uint64_t>(nkv) * 128, static_cast<uint64_t>(nkv) * 128);
  if (rc) return rc;
  rc = make_tmap_f32_scales(&tmSQ, qk_scale, Lq, 2 * static_cast<uint64_t>(heads), lds);
  if (rc) return rc;
  rc = make_tmap_f32_scales(&tmSK, qk_scale, Lk, 2 * static_cast<uint64_t>(heads), lds);
  if (rc) return rc;

  Att8Params p;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.ldo = ldo;
  p.Lq = Lq;
  p.Lk = Lk;
  p.heads = heads;
  p.nkv = nkv;
  p.v_scale = static_cast<const float*>(v_scale);
  p.scale_log2 = scale * 1.4426950408889634f;
  p.nq = (Lq + 255) / 256;
  p.ws_o = p.ws_ml = nullptr;
  // the bf16 kernel's work decomposition and workspace: yb_attention_plan / yb_attention_workspace_bytes serve both kernels
  int plan[4];
  if (int e = yb_attention_plan(Lq, Lk, heads, sm_count(), flags, plan)) return e;
  p.full_units = plan[0];
  int tail = plan[1];
  p.ns = plan[2];
  if (tail > 0) {
    const long long need = yb_attention_workspace_bytes(Lq, Lk, heads, sm_count(), flags);
    if (!ws || ws_bytes < need || (reinterpret_cast<uintptr_t>(ws) & 0xF)) {
      p.full_units += tail;   // workspace too small: run unsplit (same result, a partially filled last wave)
      tail = 0;
      p.ns = 1;
    } else {
      p.ws_o = static_cast<float*>(ws);
      p.ws_ml = p.ws_o + static_cast<size_t>(tail) * p.ns * 256 * 128;
    }
  }
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int grid = p.full_units + tail * p.ns;
  if (sp) {
    static bool attr_set[kMaxDevices] = {false};
    if (int e = ensure_dynamic_smem(attention_fp8_sp_kernel, A8_SMEM_BYTES, attr_set, "attention_fp8_sp")) return e;
    attention_fp8_sp_kernel<<<grid, A8_THREADS, A8_SMEM_BYTES, stream>>>(tmQ, tmK, tmV, tmSQ, tmSK, p, *sp);
    rc = check_launch("attention_fp8_sp");
  } else {
    static bool attr_set[kMaxDevices] = {false};
    if (int e = ensure_dynamic_smem(attention_fp8_kernel, A8_SMEM_BYTES, attr_set, "attention_fp8")) return e;
    attention_fp8_kernel<<<grid, A8_THREADS, A8_SMEM_BYTES, stream>>>(tmQ, tmK, tmV, tmSQ, tmSK, p);
    rc = check_launch("attention_fp8");
  }
  if (rc || tail == 0) return rc;
  if (sp)
    return attention_combine_launch(p.out, p.ldo, Lq, p.nq, p.full_units, p.ns, tail, p.ws_o, p.ws_ml, stream,
                                    reinterpret_cast<void* const*>(sp->out), sp->world, sp->rank, sp->Lp);
  return attention_combine_launch(p.out, p.ldo, Lq, p.nq, p.full_units, p.ns, tail, p.ws_o, p.ws_ml, stream);
}

}  // namespace yb

extern "C" int yb_attention_fp8(const void* q8, long long ldq, const void* k8, long long ldk, const void* qk_scale, long long lds,
                                const void* vt8, const void* v_scale, void* out, long long ldo, int Lq, int Lk, int heads,
                                float scale, int flags, void* ws, long long ws_bytes, void* stream_) {
  return yb::launch_attention_fp8(q8, ldq, k8, ldk, qk_scale, lds, vt8, v_scale, out, ldo, Lq, Lk, heads, scale, flags, ws,
                                  ws_bytes, nullptr, stream_);
}

extern "C" int yb_attention_fp8_sp(const void* q8, long long ldq, const void* k8, long long ldk, const void* qk_scale,
                                   long long lds, const void* vt8, const void* v_scale, void* const* out_peers, long long ldo,
                                   int Lq, int Lk, int heads, float scale, int world, int rank, int Lp, int flags, void* ws,
                                   long long ws_bytes, void* stream_) {
  using namespace yb;
  if (!out_peers || world < 2 || world > 8 || rank < 0 || rank >= world || Lp <= 0) return YB_ERR_ARG;
  if (Lq != world * Lp || Lk > Lq) return YB_ERR_ARG;
  Att8Peers sp = {};
  for (int i = 0; i < world; ++i) {
    if (!out_peers[i]) return YB_ERR_ARG;
    if (reinterpret_cast<uintptr_t>(out_peers[i]) & 0xF) return YB_ERR_ALIGNMENT;
    sp.out[i] = static_cast<__nv_bfloat16*>(out_peers[i]);
  }
  sp.world = world;
  sp.rank = rank;
  sp.Lp = Lp;
  return launch_attention_fp8(q8, ldq, k8, ldk, qk_scale, lds, vt8, v_scale, out_peers[rank], ldo, Lq, Lk, heads, scale, flags,
                              ws, ws_bytes, &sp, stream_);
}
