// attention.cu — FlashAttention-style forward for sm_90a (H100): TMA-staged Q/K/V tiles, wgmma with fp32 accumulators in
// registers, online softmax in registers, P fed back to the tensor core from registers (or shared memory, variant 1).
//
// Replaces flash_attention(q, k, v, k_lens) as used by WanSelfAttention / WanCrossAttention
// (reference: wan23/modules/attention.py:24-130 -> flash_attn_varlen_func; call sites
//  wan23/modules/model.py:197-202 self, :227 cross; wan/modules/model.py:306-311, 380-383).
// Contract kept: non-causal, softmax scale 1/sqrt(D), keys >= k_len dropped, bf16 inputs, fp32 accumulate,
// output in [L, heads, D] layout (so the o-projection GEMM reads it directly). Batch is 1 on every Yume path.
//
// CTA = one work unit of 256 query rows of one head, run as two 128-row query tiles one after the other. 384 threads:
//   warpgroup 0     TMA producer (one thread): Q tile, then K_j / V_j through an smem ring
//   warpgroups 1-2  query rows [64*(wg-1), +64) of the current tile: S = Q K_j^T (wgmma, both operands in smem), masking and
//                   online softmax on the accumulator fragment, O += P V_j with P as the register A operand
//
// Consumer schedule (FlashAttention-3's intra-warpgroup overlap), per query tile of nkv KV tiles:
//   prologue   issue S_0, wait, softmax(S_0) in place, pack P_0
//   step j     O *= alpha_j; issue S_{j+1} (not on the last step); issue O += P_j V_j;
//              wait<1> (S_{j+1} retired) -> softmax(S_{j+1}) in place, while P_j V_j runs on the tensor core;
//              wait<0> -> pack P_{j+1} (pa / the smem P were P_j V_j's operand until then)
// Every value goes through the same operations in the same order as a serial schedule (same exp2 arguments, l and O
// rescaled before the tile's terms are added, same MMA order), so the output is bit-identical to it. The softmax runs in
// place on S and is packed only after P V retires, so O + S + P = 160 registers are live, not the 224 of keeping S_j and
// S_{j+1} at once. Variant 1 (P_SMEM, a debug form) shares this schedule. ptxas would otherwise hoist wait<0> above the
// softmax; a never-taken shared store that depends on l keeps it in place (checked in the SASS: all 66 MUFU.EX2 of a step
// lie between WARPGROUP.DEPBAR.LE 1 and 0).
//
// Barriers (counts are arrivals per phase; the producer and both consumer warpgroups take ring slot it % NS and parity
// (it / NS) & 1 from one global sequence it: K_j of query tile X at it, V_j at it + 1, 2 nkv positions per tile):
//   q_full        1 + 32 KB tx  producer arrives; TMA completes      consumers wait, parity X
//   q_empty       8             each consumer warp once per tile,    producer waits before reloading Q (X = 1)
//                               after the tile's last S retired
//   kv_full[s]    1 + 32 KB tx  producer arrives; TMA completes      consumers wait: K_{j+1} before its S, V_j before P V
//   kv_empty[s]   8             each consumer warp: K_0 after the    producer waits before refilling slot s
//                               prologue, K_{j+1} after wait<1>,
//                               V_j after wait<0>
//   named 1 + wg  128           P_SMEM only: the 4 warps of warpgroup wg, before overwriting and after writing its P
// A warpgroup holds at most V_j and K_{j+1} (positions it + 1, it + 2) when it waits for K_{j+1}, having released everything
// up to it; the producer can fill it + 2 once it + 2 - NS <= it is released, so any NS >= 2 is deadlock-free (5 slots, 4 with
// P_SMEM). Any nkv >= 1 works, so the last, shorter KV segment of the tail split needs nothing special.
//
// Tail split: a launch is U = heads x ceil(Lq/256) equal work units. When the last wave is at most half full its T units are each
// cut into ns KV segments that run as separate CTAs and leave (unnormalised O, row max, row sum) in a workspace; a small combine
// kernel merges the segments and performs the normal epilogue (bf16 store / Ulysses peer scatter).
#include "yb_host.h"
#include "yb_ptx.cuh"

namespace yb {

constexpr int ATT_THREADS = 384;
constexpr int ATT_TILE_BYTES = 128 * 128 * 2;  // one 128x128 bf16 tile = 2 swizzled slabs of 16 KB

struct AttParams {
  __nv_bfloat16* out;
  long long ldo;
  int Lq, Lk;
  int nkv;
  int accumulate;    // out += result (sum of two attention branches)
  // Ulysses (sp_world > 1): output row g belongs to rank g / sp_Lp and is stored straight into that rank's
  // [P(src), Lp, heads_local*128] receive buffer over NVLink (peer pointers) — the all-to-all is the epilogue itself.
  __nv_bfloat16* out_peers[8];
  int sp_world, sp_rank, sp_Lp;
  float scale_log2;  // softmax scale * log2(e)
  // work decomposition: unit u = head * nq + q_block. CTAs [0, full_units) run whole units; CTA full_units + r runs KV
  // segment r % ns of unit full_units + r / ns and writes a partial result to the workspace
  int nq, full_units, ns;
  float* ws_o;       // [tail CTAs, 256, 128] unnormalised O
  float* ws_ml;      // [tail CTAs, 256, 2]   (row max in the log2 domain, row sum)
};

template <bool P_SMEM>
struct AttCfg {
  static constexpr int NS = P_SMEM ? 4 : 5;  // KV ring slots
  static constexpr int Q_OFF = 0;
  static constexpr int P_OFF = ATT_TILE_BYTES;   // P_SMEM: 64 x 128 bf16 per consumer warpgroup (2 slabs of 8 KB)
  static constexpr int KV_OFF = P_SMEM ? 2 * ATT_TILE_BYTES : ATT_TILE_BYTES;
  static constexpr int BAR_OFF = KV_OFF + NS * ATT_TILE_BYTES;
  static constexpr int SINK_OFF = BAR_OFF + 128;   // a word no one reads (see the wait after the softmax)
  static_assert((2 + 2 * NS) * 8 <= 128, "mbarriers below the sink word");
  static constexpr int SMEM_BYTES = BAR_OFF + 256 + 1024;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
};

template <bool P_SMEM>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const AttParams p) {
  using Cfg = AttCfg<P_SMEM>;
  constexpr int NS = Cfg::NS;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + Cfg::BAR_OFF);
  uint64_t* q_empty = q_full + 1;
  uint64_t* kv_full = q_empty + 1;
  uint64_t* kv_empty = kv_full + NS;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // work decomposition (see AttParams)
  int unit = blockIdx.x, kv_begin = 0, nkv = p.nkv;
  if (static_cast<int>(blockIdx.x) >= p.full_units) {  // KV segment of a tail unit
    const int r = blockIdx.x - p.full_units;
    unit = p.full_units + r / p.ns;
    const int per = (((p.nkv + p.ns - 1) / p.ns) + 1) & ~1;
    kv_begin = (r % p.ns) * per;
    nkv = min(per, p.nkv - kv_begin);
  }
  const int head = unit / p.nq;
  const int q0 = (unit - head * p.nq) * 256;
  const int nx = q0 + 128 < p.Lq ? 2 : 1;   // query tiles of this unit that hold rows < Lq

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    mbar_init(q_empty, 8);
    for (int i = 0; i < NS; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 8);   // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      // ------------------------------- TMA producer -------------------------------
      int it = 0;
      for (int X = 0; X < nx; ++X) {
        if (X == 1) mbar_wait(q_empty, 0);
        mbar_arrive_expect_tx(q_full, ATT_TILE_BYTES);
        for (int s = 0; s < 2; ++s)
          tma_load_2d(smem + Cfg::Q_OFF + s * 16384, &tmQ, q_full, head * 128 + s * 64, q0 + X * 128);
        for (int jj = 0; jj < 2 * nkv; ++jj, ++it) {
          const int slot = it % NS;
          mbar_wait(&kv_empty[slot], ((it / NS) & 1) ^ 1);
          mbar_arrive_expect_tx(&kv_full[slot], ATT_TILE_BYTES);
          const CUtensorMap* tm = (jj & 1) ? &tmV : &tmK;
          uint8_t* dst = smem + Cfg::KV_OFF + slot * ATT_TILE_BYTES;
          const int j = kv_begin + (jj >> 1);
          tma_load_2d(dst, tm, &kv_full[slot], head * 128, j * 128);
          tma_load_2d(dst + 16384, tm, &kv_full[slot], head * 128 + 64, j * 128);
        }
      }
    }
  } else {
    // ------------------------------- S, softmax, P V, epilogue -------------------------------
    setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;
    const int q4 = lane >> 2, c2 = 2 * (lane & 3);   // fragment rows q4 / q4 + 8 of the warp's 16, columns 8g + c2, +1
    const int row_a = wg * 64 + (warp & 3) * 16 + q4;   // tile row of fragment row a (row b = row_a + 8)
    const float sc = p.scale_log2;
    const uint32_t sQ = smem_u32(smem + Cfg::Q_OFF) + wg * 64 * 128;
    const uint32_t sP = smem_u32(smem + Cfg::P_OFF) + wg * 16384;
    // S = Q K^T of the K tile at ring position `itk`, committed as one wgmma group and not waited for. s is not zeroed: the
    // first k-step overwrites it.
    auto issue_s = [&](float (&s)[64], int itk) {
      const int slot_k = itk % NS;
      att_wait(&kv_full[slot_k], (itk / NS) & 1);
      const uint32_t sK = smem_u32(smem + Cfg::KV_OFF + slot_k * ATT_TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {   // D = 128: two 64-column slabs, 4 k-steps of 32 B each
        const uint32_t off = (kk >> 2) * 16384 + (kk & 3) * 32;
        wgmma_ss_acc64<0>(s, make_smem_desc_sw128(sQ + off, 16, 1024), make_smem_desc_sw128(sK + off, 16, 1024), kk != 0);
      }
      wgmma_commit();
    };
    int it = 0;
    for (int X = 0; X < nx; ++X) {
      att_wait(q_full, X);
      float o[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) o[i] = 0.f;
      float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows a / b: running max (log2 domain) and sum
      float al0, al1;      // rescale factors of O for the tile whose P is in pa
      float s[64];         // S of one KV tile, overwritten in place by its exponentials
      uint32_t pa[8][4];   // P as the A fragment of the k-steps of P V: k-step kk covers keys [16kk, 16kk + 16)
      // Online softmax of KV tile j on s: mask, row max, rescale factors, l, and the exponentials in place. O is left to
      // the caller, which rescales it by al0 / al1 right before the P V of this tile.
      auto softmax = [&](int j) {
        const int kv_rem = p.Lk - (kv_begin + j) * 128;
        if (kv_rem < 128) {   // last, partial KV tile (k_lens contract): columns past the end count as -inf
#pragma unroll
          for (int i = 0; i < 64; ++i)
            if (8 * (i >> 2) + c2 + (i & 1) >= kv_rem) s[i] = -INFINITY;
        }
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
        const float mn0 = fmaxf(m0, mx0 * sc), mn1 = fmaxf(m1, mx1 * sc);
        al0 = fast_exp2(m0 - mn0);   // 0 on the first tile (m = -inf)
        al1 = fast_exp2(m1 - mn1);
        m0 = mn0;
        m1 = mn1;
        l0 *= al0;
        l1 *= al1;
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {   // accumulator groups 2kk, 2kk + 1
          float* e = s + 8 * kk;
#pragma unroll
          for (int i = 0; i < 8; ++i) e[i] = fast_exp2(e[i] * sc - ((i & 2) ? m1 : m0));
          l0 += (e[0] + e[1]) + (e[4] + e[5]);
          l1 += (e[2] + e[3]) + (e[6] + e[7]);
        }
      };
      // exponentials of s -> bf16 P (registers, or this warpgroup's shared-memory P for variant 1)
      auto pack_p = [&]() {
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
          const float* e = s + 8 * kk;
          pa[kk][0] = pack_bf16x2(e[0], e[1]);   // row a, keys 2t, 2t+1
          pa[kk][1] = pack_bf16x2(e[2], e[3]);   // row b
          pa[kk][2] = pack_bf16x2(e[4], e[5]);   // row a, keys 8 + 2t, +1
          pa[kk][3] = pack_bf16x2(e[6], e[7]);   // row b
        }
        if (P_SMEM) {
          named_bar_sync(1 + wg, 128);   // every warp's wait for the previous P V is over: P may be overwritten
          // K-major 128B-swizzled P of this warpgroup: slab = key / 64; row r, 16-byte chunk c -> r*128 + ((c ^ (r & 7)) << 4)
          const int ra = row_a - wg * 64, rb = ra + 8;
#pragma unroll
          for (int kk = 0; kk < 8; ++kk) {
            uint8_t* slab = smem + Cfg::P_OFF + wg * 16384 + (kk >> 2) * 8192;
            const int k0 = (kk & 3) * 16 + c2, k1 = k0 + 8;   // key within the slab
            *reinterpret_cast<uint32_t*>(slab + ra * 128 + (((k0 >> 3) ^ (ra & 7)) << 4) + (k0 & 7) * 2) = pa[kk][0];
            *reinterpret_cast<uint32_t*>(slab + rb * 128 + (((k0 >> 3) ^ (rb & 7)) << 4) + (k0 & 7) * 2) = pa[kk][1];
            *reinterpret_cast<uint32_t*>(slab + ra * 128 + (((k1 >> 3) ^ (ra & 7)) << 4) + (k1 & 7) * 2) = pa[kk][2];
            *reinterpret_cast<uint32_t*>(slab + rb * 128 + (((k1 >> 3) ^ (rb & 7)) << 4) + (k1 & 7) * 2) = pa[kk][3];
          }
          fence_proxy_async_smem();
          named_bar_sync(1 + wg, 128);
        }
      };

      issue_s(s, it);   // prologue: S_0, its softmax and P_0, with nothing to overlap
      wgmma_wait<0>();
      fence_regs(s);
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&kv_empty[it % NS]);
        if (nkv == 1) mbar_arrive(q_empty);   // that was the tile's last S: the producer may reload Q
      }
      softmax(0);
      pack_p();
      // KV tile j: P_j is packed and al0 / al1 are its rescale factors (see the schedule in the header). The last tile is a
      // separate call with next = false so that every wgmma group and wait is unconditional within a call: with a runtime
      // condition around the S issue and its wait, ptxas serialises every wgmma of the kernel.
      auto kv_step = [&](int j, const bool next) {
        const int slot_v = (it + 1) % NS, slot_kn = (it + 2) % NS;
#pragma unroll
        for (int g = 0; g < 16; ++g) {   // before the first wgmma of the step: ptxas serialises a stage whose accumulators
          o[4 * g] *= al0;               // are touched between its wgmmas
          o[4 * g + 1] *= al0;
          o[4 * g + 2] *= al1;
          o[4 * g + 3] *= al1;
        }
        if (next) issue_s(s, it + 2);
        att_wait(&kv_full[slot_v], ((it + 1) / NS) & 1);
        const uint32_t sV = smem_u32(smem + Cfg::KV_OFF + slot_v * ATT_TILE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {   // V is MN-major: 16 keys = 2048 B further, D slabs 16 KB apart
          const uint64_t vdesc = make_smem_desc_sw128(sV + kk * 2048, 16384, 1024);
          if (P_SMEM)
            wgmma_ss_acc64<1>(o, make_smem_desc_sw128(sP + (kk >> 2) * 8192 + (kk & 3) * 32, 16, 1024), vdesc, 1u);
          else
            wgmma_rs_n128_tb(o, pa[kk], vdesc, 1u);
        }
        wgmma_commit();
        if (next) {
          wgmma_wait<1>();   // groups retire in order: S_{j+1} is done, P_j V_j may still run
          fence_regs(s);
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(&kv_empty[slot_kn]);
            if (j + 2 == nkv) mbar_arrive(q_empty);
          }
          softmax(j + 1);
          // ptxas schedules wgmma.wait_group freely among register arithmetic and would hoist the wait below above the
          // softmax, leaving nothing to overlap P_j V_j. It keeps the wait after shared-memory accesses, so a store that
          // depends on every exponential (through l) and is never taken (l >= 0) pins the softmax ahead of the wait.
          if (l0 + l1 < 0.f) *reinterpret_cast<volatile float*>(smem + Cfg::SINK_OFF) = l0;
        }
        wgmma_wait<0>();
        fence_regs(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(&kv_empty[slot_v]);
        if (next) pack_p();   // pa / the shared-memory P were P_j V_j's operand until now
        it += 2;
      };
      for (int j = 0; j + 1 < nkv; ++j) kv_step(j, true);
      kv_step(nkv - 1, false);
      l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
      l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 2);

      // epilogue: O / l -> bf16 -> global [Lq, heads*128] (or the KV-segment workspace / the owner rank's receive buffer)
#pragma unroll
      for (int h = 0; h < 2; ++h) {   // fragment row a, then row b
        const int row_t = X * 128 + row_a + 8 * h;
        const float m = h ? m1 : m0, l = h ? l1 : l0;
        if (static_cast<int>(blockIdx.x) >= p.full_units) {
          const long long prow = static_cast<long long>(blockIdx.x - p.full_units) * 256 + row_t;
          float* wo = p.ws_o + prow * 128;
#pragma unroll
          for (int g = 0; g < 16; ++g) *reinterpret_cast<float2*>(wo + 8 * g + c2) = make_float2(o[4 * g + 2 * h], o[4 * g + 2 * h + 1]);
          if ((lane & 3) == 0) *reinterpret_cast<float2*>(p.ws_ml + prow * 2) = make_float2(m, l);
          continue;
        }
        const int q_row = q0 + row_t;
        if (q_row >= p.Lq) continue;
        __nv_bfloat16* orow = p.out + static_cast<long long>(q_row) * p.ldo + head * 128;
        if (p.sp_world > 1) {
          const int owner = q_row / p.sp_Lp;
          const int t = q_row - owner * p.sp_Lp;
          if (owner < p.sp_world)
            orow = p.out_peers[owner] + (static_cast<long long>(p.sp_rank) * p.sp_Lp + t) * p.ldo + head * 128;
        }
        const float inv = 1.0f / l;
#pragma unroll
        for (int g = 0; g < 16; ++g) {
          uint32_t* dst = reinterpret_cast<uint32_t*>(orow + 8 * g + c2);
          float v0 = o[4 * g + 2 * h] * inv, v1 = o[4 * g + 2 * h + 1] * inv;
          if (p.accumulate) {
            const float2 prev = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(dst));
            v0 += prev.x;
            v1 += prev.y;
          }
          *dst = pack_bf16x2(v0, v1);
        }
      }
    }
  }
}

// Merge the ns KV-segment partials of every tail unit and do the normal epilogue. One warp per query row, 4 columns per
// lane: out = sum_s O_s 2^(m_s - M) / sum_s l_s 2^(m_s - M).
__global__ void __launch_bounds__(256) attention_combine_kernel(const AttParams p, int tail_units) {
  const int gw = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (gw >= tail_units * 256) return;
  const int tu = gw >> 8, r = gw & 255;
  const int unit = p.full_units + tu;
  const int head = unit / p.nq;
  const int q_row = (unit - head * p.nq) * 256 + r;
  if (q_row >= p.Lq) return;
  float M = -INFINITY;
  for (int sgm = 0; sgm < p.ns; ++sgm) M = fmaxf(M, p.ws_ml[((static_cast<long long>(tu) * p.ns + sgm) * 256 + r) * 2]);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float lsum = 0.f;
  for (int sgm = 0; sgm < p.ns; ++sgm) {
    const long long prow = (static_cast<long long>(tu) * p.ns + sgm) * 256 + r;
    const float2 ml = *reinterpret_cast<const float2*>(p.ws_ml + prow * 2);
    const float w = exp2f(ml.x - M);
    const float4 o = *reinterpret_cast<const float4*>(p.ws_o + prow * 128 + lane * 4);
    acc.x += o.x * w; acc.y += o.y * w; acc.z += o.z * w; acc.w += o.w * w;
    lsum += ml.y * w;
  }
  const float inv = 1.0f / lsum;
  __nv_bfloat16* orow = p.out + static_cast<long long>(q_row) * p.ldo + head * 128;
  if (p.sp_world > 1) {
    const int owner = q_row / p.sp_Lp;
    const int t = q_row - owner * p.sp_Lp;
    if (owner < p.sp_world)
      orow = p.out_peers[owner] + (static_cast<long long>(p.sp_rank) * p.sp_Lp + t) * p.ldo + head * 128;
  }
  *reinterpret_cast<uint2*>(orow + lane * 4) = make_uint2(pack_bf16x2(acc.x * inv, acc.y * inv), pack_bf16x2(acc.z * inv, acc.w * inv));
}

// Work decomposition of one launch (pure host arithmetic; exported as yb_attention_plan for the CPU test-suite).
//   units        heads x ceil(Lq / 256) equal work units
//   force_ns     0 = automatic, 1 = never split, 2..4 = split every unit into that many KV segments
// Automatic rule: when the last wave on `sms` SMs is at most half full and there is more than one wave, its `tail` units
// are cut into ns = min(4, sms / tail) KV segments. Segment length is rounded up to an EVEN number of 128-key tiles (the
// kernel takes barrier parities from the global tile index) and every segment must own at least one tile.
static void attention_plan(int units, int nkv, int sms, bool allowed, int force_ns, int* full_units, int* tail, int* ns) {
  *full_units = units;
  *tail = 0;
  *ns = 1;
  if (!allowed || force_ns == 1) return;
  if (force_ns >= 2 && nkv >= 2 * force_ns) {
    *tail = units;
    *ns = force_ns;
  } else if (force_ns == 0 && units > sms && units % sms != 0 && 2 * (units % sms) <= sms && nkv >= 16) {
    *tail = units % sms;
    *ns = sms / *tail < 4 ? sms / *tail : 4;
  }
  while (*ns > 1 && (*ns - 1) * ((((nkv + *ns - 1) / *ns) + 1) & ~1) >= nkv) --*ns;
  if (*ns == 1) *tail = 0;
  *full_units = units - *tail;
}

// Workspace of the tail split: tail CTAs x 256 rows x (128 + 2) floats, CALLER-owned (the library never allocates and never
// synchronises: yb_attention_workspace_bytes sizes it). Without a large enough workspace the launch is simply not split.
static size_t split_workspace_bytes(size_t ctas) { return ctas * 256 * 130 * sizeof(float); }

static int g_debug_force_split = 0;   // yb_debug_force_split: tests force the KV split through paths that carry no flags

// force_ns: 0 = automatic tail split, 1 = never, 2..4 = split EVERY unit into that many KV segments (tests)
template <bool P_SMEM>
static int launch_attention(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                            AttParams p, int heads, cudaStream_t stream, int force_ns, void* ws, long long ws_bytes) {
  using Cfg = AttCfg<P_SMEM>;
  auto kern = attention_kernel<P_SMEM>;
  static bool attr_set[kMaxDevices] = {false};
  if (int rc = ensure_dynamic_smem(kern, Cfg::SMEM_BYTES, attr_set, "attention")) return rc;
  if (force_ns == 0 && g_debug_force_split >= 1 && g_debug_force_split <= 4) force_ns = g_debug_force_split;
  p.nq = (p.Lq + 255) / 256;
  const int units = p.nq * heads;
  int tail = 0;
  p.ws_o = p.ws_ml = nullptr;
  const bool allowed = !p.accumulate && ws != nullptr;
  attention_plan(units, p.nkv, sm_count(), allowed, force_ns, &p.full_units, &tail, &p.ns);
  if (tail > 0) {
    const size_t ctas = static_cast<size_t>(tail) * p.ns;
    if (ws_bytes < 0 || static_cast<size_t>(ws_bytes) < split_workspace_bytes(ctas) || (reinterpret_cast<uintptr_t>(ws) & 0xF)) {
      p.full_units = units;   // workspace too small: run unsplit (same result, a partially filled last wave)
      tail = 0;
      p.ns = 1;
    } else {
      p.ws_o = static_cast<float*>(ws);
      p.ws_ml = p.ws_o + ctas * 256 * 128;
    }
  }
  kern<<<p.full_units + tail * p.ns, ATT_THREADS, Cfg::SMEM_BYTES, stream>>>(tmQ, tmK, tmV, p);
  int rc = check_launch("attention");
  if (rc || tail == 0) return rc;
  attention_combine_kernel<<<tail * 32, 256, 0, stream>>>(p, tail);
  return check_launch("attention_combine");
}

// the combine for another attention kernel that writes its KV-segment partials in this layout (attention_fp8.cu)
int attention_combine_launch(void* out, long long ldo, int Lq, int nq, int full_units, int ns, int tail, float* ws_o,
                             float* ws_ml, cudaStream_t stream, void* const* out_peers, int world, int rank, int Lp) {
  AttParams p = {};
  p.out = static_cast<__nv_bfloat16*>(out);
  p.ldo = ldo;
  p.Lq = Lq;
  p.sp_world = out_peers ? world : 1;
  if (out_peers) {
    for (int i = 0; i < 8; ++i) p.out_peers[i] = i < world ? static_cast<__nv_bfloat16*>(out_peers[i]) : nullptr;
    p.sp_rank = rank;
    p.sp_Lp = Lp;
  }
  p.nq = nq;
  p.full_units = full_units;
  p.ns = ns;
  p.ws_o = ws_o;
  p.ws_ml = ws_ml;
  attention_combine_kernel<<<tail * 32, 256, 0, stream>>>(p, tail);
  return check_launch("attention_combine");
}

// debug variant (P through shared memory) selected by flags bit 0
static int dispatch_attention(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                              AttParams p, int heads, cudaStream_t stream, int flags, void* ws, long long ws_bytes) {
  const int force_ns = (flags >> YB_ATT_SPLIT_SHIFT) & 7;
  if (force_ns > 4) return YB_ERR_ARG;
  if ((flags >> YB_ATT_EMU_SHIFT) & 3) return YB_ERR_ARG;   // retired: FMA-pipe exponentials (measured slower, removed)
  CUtensorMap tmQ, tmK, tmV;
  const uint64_t cols = static_cast<uint64_t>(heads) * 128;
  int rc = make_tmap_bf16_2d(&tmQ, q, p.Lq, cols, ldq, 128, 64);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmK, k, p.Lk, cols, ldk, 128, 64);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmV, v, p.Lk, cols, ldv, 128, 64);
  if (rc) return rc;
  if (flags & YB_ATT_P_SMEM) return launch_attention<true>(tmQ, tmK, tmV, p, heads, stream, force_ns, ws, ws_bytes);
  return launch_attention<false>(tmQ, tmK, tmV, p, heads, stream, force_ns, ws, ws_bytes);
}

}  // namespace yb

extern "C" int yb_debug_force_split(int ns) {
  if (ns < 0 || ns > 4) return YB_ERR_ARG;
  yb::g_debug_force_split = ns;
  return YB_OK;
}

extern "C" int yb_attention_plan(int Lq, int Lk, int heads, int sms, int flags, int* out4) {
  if (Lq <= 0 || Lk <= 0 || heads <= 0 || sms <= 0 || !out4) return YB_ERR_ARG;
  int force_ns = (flags >> YB_ATT_SPLIT_SHIFT) & 7;
  if (force_ns > 4) return YB_ERR_ARG;
  if (force_ns == 0 && yb::g_debug_force_split >= 1) force_ns = yb::g_debug_force_split;
  const int nkv = (Lk + 127) / 128;
  int full_units, tail, ns;
  yb::attention_plan(((Lq + 255) / 256) * heads, nkv, sms, !(flags & YB_ATT_ACCUMULATE), force_ns, &full_units, &tail, &ns);
  out4[0] = full_units;
  out4[1] = tail;
  out4[2] = ns;
  out4[3] = ns > 1 ? ((((nkv + ns - 1) / ns) + 1) & ~1) : nkv;   // KV tiles per segment
  return YB_OK;
}

extern "C" long long yb_attention_workspace_bytes(int Lq, int Lk, int heads, int sms, int flags) {
  int plan[4];
  if (yb_attention_plan(Lq, Lk, heads, sms, flags, plan)) return -1;
  return static_cast<long long>(yb::split_workspace_bytes(static_cast<size_t>(plan[1]) * plan[2]));
}

extern "C" int yb_attention_ex(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                               long long ldv, void* out, long long ldo, int Lq, int Lk, int heads, float scale,
                               int flags, void* ws, long long ws_bytes, void* trace, void* stream_) {
  using namespace yb;
  if (!q || !k || !v || !out) return YB_ERR_ARG;
  if (Lq <= 0 || Lk <= 0 || heads <= 0) return YB_ERR_ARG;
  if ((ldo % 8) != 0 || (reinterpret_cast<uintptr_t>(out) & 0xF)) return YB_ERR_ALIGNMENT;
  AttParams p;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.ldo = ldo;
  p.Lq = Lq;
  p.Lk = Lk;
  p.nkv = (Lk + 127) / 128;
  p.accumulate = (flags & YB_ATT_ACCUMULATE) ? 1 : 0;
  (void)trace;   // accepted for ABI compatibility, ignored (see include/yume_b200.h)
  p.sp_world = 1;
  p.sp_rank = 0;
  p.sp_Lp = 0;
  p.scale_log2 = scale * 1.4426950408889634f;
  return dispatch_attention(q, ldq, k, ldk, v, ldv, p, heads, reinterpret_cast<cudaStream_t>(stream_), flags, ws, ws_bytes);
}

extern "C" int yb_attention(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                            void* out, long long ldo, int Lq, int Lk, int heads, float scale, int flags,
                            void* stream_) {
  return yb_attention_ex(q, ldq, k, ldk, v, ldv, out, ldo, Lq, Lk, heads, scale, flags, nullptr, 0, nullptr, stream_);
}

// Ulysses attention: same kernel, output rows scattered to their owner ranks through peer pointers (see AttParams).
extern "C" int yb_attention_sp(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                               void* const* out_peers, long long ldo, int Lq, int Lk, int heads, float scale, int world,
                               int rank, int Lp, int flags, void* ws, long long ws_bytes, void* stream_) {
  using namespace yb;
  if (!q || !k || !v || !out_peers || world < 2 || world > 8 || rank < 0 || rank >= world || Lp <= 0) return YB_ERR_ARG;
  if (Lq != world * Lp || Lk <= 0 || Lk > Lq || heads <= 0 || (ldo % 8)) return YB_ERR_ARG;
  if (flags & (YB_ATT_ACCUMULATE | YB_ATT_P_SMEM)) return YB_ERR_ARG;
  AttParams p;
  p.out = static_cast<__nv_bfloat16*>(out_peers[rank]);
  p.ldo = ldo;
  p.Lq = Lq;
  p.Lk = Lk;
  p.nkv = (Lk + 127) / 128;
  p.accumulate = 0;
  p.scale_log2 = scale * 1.4426950408889634f;
  for (int i = 0; i < 8; ++i) p.out_peers[i] = i < world ? static_cast<__nv_bfloat16*>(out_peers[i]) : nullptr;
  p.sp_world = world;
  p.sp_rank = rank;
  p.sp_Lp = Lp;
  return dispatch_attention(q, ldq, k, ldk, v, ldv, p, heads, reinterpret_cast<cudaStream_t>(stream_), flags, ws, ws_bytes);
}
