// t5.cu — the three kernels of the umT5-XXL text encoder (wan/modules/t5.py:267-312) that the DiT kernels do not cover:
// relative-position-bias attention with a key padding mask and no 1/sqrt(d) scale at head_dim 64, the T5 RMS norm (no mean,
// no bias) from the fp32 residual stream, and the gated-GELU product of the feed-forward. The projections run on yb_gemm_bf16.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "../../include/yume_b200_t5.h"
#include "yb_host.h"
#include "yb_ptx.cuh"

namespace {

typedef __nv_bfloat16 bf16;

// ------------------------------------------------------------------------------------------------
// attention
// ------------------------------------------------------------------------------------------------
constexpr int T5_HD = 64;            // head_dim
constexpr int T5_BQ = 64;            // query rows per CTA: 4 warps x 16
constexpr int T5_BK = 64;            // keys per K/V tile
constexpr int T5_LDS = T5_HD + 8;    // smem row pitch in bf16 (144 B): fragment loads and ldmatrix rows are conflict-free
constexpr int T5_THREADS = 128;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  // src-size 0 zero-fills the 16 bytes (rows past L): masked keys then meet P = 0 against V = 0, never garbage
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(yb::smem_u32(smem)), "l"(gmem), "r"(valid ? 16 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

// D (16 x 8, f32) += A (16 x 16, bf16, row) * B (16 x 8, bf16, col). Fragments of lane (g = lane / 4, t = lane % 4):
// a = {A[g][2t..], A[g+8][2t..], A[g][2t+8..], A[g+8][2t+8..]}, b = {B[2t..][g], B[2t+8..][g]},
// d = {D[g][2t], D[g][2t+1], D[g+8][2t], D[g+8][2t+1]}.
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(yb::smem_u32(smem))
               : "memory");
}

__device__ __forceinline__ uint32_t lds32(const bf16* p) { return *reinterpret_cast<const uint32_t*>(p); }

// One CTA per (64-query tile, head, sample); warp w owns query rows 16w .. 16w+15 of the tile. The Q tile and the first two
// K/V tiles are fetched with cp.async, then K/V tiles of 64 keys stream through a double buffer with an online softmax:
//   S = Q K^T (fp32, mma.sync) + bias[h, j - i + L - 1]; keys j >= L or key_mask[b, j] == 0 are dropped (-inf);
//   m' = max(m, rowmax S); alpha = exp(m - m'); l = l*alpha + sum exp(S - m'); O = O*alpha + bf16(exp(S - m')) V.
// The exponentials are __expf (ex2.approx of x*log2(e)); P is the fp32 S fragment packed to bf16 in registers, which is the
// A fragment of the P.V mma; V's B fragments come from ldmatrix.trans. out = O / l rounded to bf16 (0 for a row whose every
// key is masked).
__global__ void __launch_bounds__(T5_THREADS)
t5_attention_kernel(const bf16* __restrict__ q, long long ldq, const bf16* __restrict__ k, long long ldk,
                    const bf16* __restrict__ v, long long ldv, bf16* __restrict__ out, long long ldo, int L,
                    const float* __restrict__ bias, const unsigned char* __restrict__ key_mask) {
  __shared__ __align__(16) bf16 sQ[T5_BQ * T5_LDS];
  __shared__ __align__(16) bf16 sK[2][T5_BK * T5_LDS];
  __shared__ __align__(16) bf16 sV[2][T5_BK * T5_LDS];
  const int h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const long long row0 = static_cast<long long>(b) * L;
  const int q0 = blockIdx.x * T5_BQ;
  const int nkv = (L + T5_BK - 1) / T5_BK;

  auto load_tile = [&](bf16* dst, const bf16* src, long long ld, int r0) {
    for (int c = tid; c < 64 * 8; c += T5_THREADS) {            // 64 rows x 8 chunks of 16 B
      const int r = c >> 3, ch = c & 7;
      const bool valid = r0 + r < L;
      const bf16* p = valid ? src + (row0 + r0 + r) * ld + h * T5_HD + ch * 8 : src;
      cp_async16(dst + r * T5_LDS + ch * 8, p, valid);
    }
  };
  load_tile(sQ, q, ldq, q0);
  load_tile(sK[0], k, ldk, 0);
  load_tile(sV[0], v, ldv, 0);
  cp_async_commit();
  if (nkv > 1) {
    load_tile(sK[1], k, ldk, T5_BK);
    load_tile(sV[1], v, ldv, T5_BK);
  }
  cp_async_commit();

  const float* brow = bias + static_cast<long long>(h) * (2 * L - 1);
  const unsigned char* mrow = key_mask ? key_mask + row0 : nullptr;
  const int i_lo = q0 + warp * 16 + g, i_hi = i_lo + 8;       // the two query rows of this lane
  const bool ok_lo = i_lo < L, ok_hi = i_hi < L;

  uint32_t qa[4][4];
  float o[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;

  for (int j = 0; j < nkv; ++j) {
    cp_async_wait_1();                 // every group but the newest is complete: tile j (and Q) have landed
    __syncthreads();
    const int buf = j & 1;
    if (j == 0) {
      const bf16* qs = sQ + (warp * 16 + g) * T5_LDS + 2 * t;
#pragma unroll
      for (int kc = 0; kc < 4; ++kc) {
        qa[kc][0] = lds32(qs + kc * 16);
        qa[kc][1] = lds32(qs + 8 * T5_LDS + kc * 16);
        qa[kc][2] = lds32(qs + kc * 16 + 8);
        qa[kc][3] = lds32(qs + 8 * T5_LDS + kc * 16 + 8);
      }
    }
    const bf16* Ks = sK[buf];
    const bf16* Vs = sV[buf];
    float s[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
      const bf16* kr = Ks + (n * 8 + g) * T5_LDS + 2 * t;
#pragma unroll
      for (int kc = 0; kc < 4; ++kc) mma_16816(s[n], qa[kc], lds32(kr + kc * 16), lds32(kr + kc * 16 + 8));
    }
    const int kbase = j * T5_BK;
    float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int key = kbase + n * 8 + 2 * t + e;
        const bool keep = key < L && (mrow == nullptr || mrow[key] != 0);
        // rows past L are never stored: they take no bias (their bias index would leave the table)
        s[n][e] = keep ? s[n][e] + (ok_lo ? __ldg(brow + (key - i_lo + L - 1)) : 0.f) : -INFINITY;
        s[n][e + 2] = keep ? s[n][e + 2] + (ok_hi ? __ldg(brow + (key - i_hi + L - 1)) : 0.f) : -INFINITY;
        mx_lo = fmaxf(mx_lo, s[n][e]);
        mx_hi = fmaxf(mx_hi, s[n][e + 2]);
      }
    }
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
    const float mn_lo = fmaxf(m_lo, mx_lo), mn_hi = fmaxf(m_hi, mx_hi);
    const float base_lo = mn_lo == -INFINITY ? 0.f : mn_lo;     // no key kept so far: exp(-inf - 0) = 0 everywhere
    const float base_hi = mn_hi == -INFINITY ? 0.f : mn_hi;
    const float al_lo = __expf(m_lo - base_lo), al_hi = __expf(m_hi - base_hi);
    m_lo = mn_lo;
    m_hi = mn_hi;
    float sum_lo = 0.f, sum_hi = 0.f;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      s[n][0] = __expf(s[n][0] - base_lo);
      s[n][1] = __expf(s[n][1] - base_lo);
      s[n][2] = __expf(s[n][2] - base_hi);
      s[n][3] = __expf(s[n][3] - base_hi);
      sum_lo += s[n][0] + s[n][1];
      sum_hi += s[n][2] + s[n][3];
      o[n][0] *= al_lo;
      o[n][1] *= al_lo;
      o[n][2] *= al_hi;
      o[n][3] *= al_hi;
    }
    l_lo = l_lo * al_lo + sum_lo;
    l_hi = l_hi * al_hi + sum_hi;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {                           // 16 keys per k-step
      const uint32_t pa[4] = {yb::pack_bf16x2(s[2 * kk][0], s[2 * kk][1]), yb::pack_bf16x2(s[2 * kk][2], s[2 * kk][3]),
                              yb::pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]),
                              yb::pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3])};
      const bf16* vr = Vs + (kk * 16 + ((lane >> 3) & 1) * 8 + (lane & 7)) * T5_LDS + (lane >> 4) * 8;
#pragma unroll
      for (int np = 0; np < 4; ++np) {                         // 16 output columns per ldmatrix.x4
        uint32_t r[4];
        ldmatrix_x4_trans(r, vr + np * 16);
        mma_16816(o[2 * np], pa, r[0], r[1]);
        mma_16816(o[2 * np + 1], pa, r[2], r[3]);
      }
    }
    __syncthreads();                   // every warp is done with buffer `buf` before it is refilled
    if (j + 2 < nkv) {
      load_tile(sK[buf], k, ldk, (j + 2) * T5_BK);
      load_tile(sV[buf], v, ldv, (j + 2) * T5_BK);
    }
    cp_async_commit();                 // possibly empty: keeps one group per iteration for the wait above
  }

  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
  const float inv_lo = l_lo > 0.f ? 1.f / l_lo : 0.f, inv_hi = l_hi > 0.f ? 1.f / l_hi : 0.f;
  bf16* olo = out + (row0 + i_lo) * ldo + h * T5_HD + 2 * t;
  bf16* ohi = out + (row0 + i_hi) * ldo + h * T5_HD + 2 * t;
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    if (ok_lo) *reinterpret_cast<uint32_t*>(olo + n * 8) = yb::pack_bf16x2(o[n][0] * inv_lo, o[n][1] * inv_lo);
    if (ok_hi) *reinterpret_cast<uint32_t*>(ohi + n * 8) = yb::pack_bf16x2(o[n][2] * inv_hi, o[n][3] * inv_hi);
  }
}

// ------------------------------------------------------------------------------------------------
// T5 RMS norm: one warp per row, the row in registers (C = 128 * NV), shuffle-only reduction
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Read-only 16-byte load the compiler may not move (as ldg_f4_ordered in elementwise.cu): unordered, ptxas hoists all NV
// weight loads above the apply loop and the row no longer fits beside them.
__device__ __forceinline__ float4 ldg_f4_ordered(const float* p) {
  float4 v;
  asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}

template <int NV, bool OUT_F32>
__global__ void __launch_bounds__(256)
t5_rmsnorm_kernel(const float* __restrict__ x, long long ldx, void* __restrict__ out, long long ldo,
                  const float* __restrict__ weight, int L, float eps) {
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
  for (int i = 0; i < NV; ++i) s += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
  const float rstd = rsqrtf(warp_sum(s) / static_cast<float>(C) + eps);
  const float* wp = weight + lane * 4;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float4 w = ldg_f4_ordered(wp + i * 128);
    float4 y;
    y.x = (v[i].x * rstd) * w.x;
    y.y = (v[i].y * rstd) * w.y;
    y.z = (v[i].z * rstd) * w.z;
    y.w = (v[i].w * rstd) * w.w;
    const int idx = lane + i * 32;
    if (OUT_F32) {
      reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + static_cast<long long>(row) * ldo)[idx] = y;
    } else {
      uint2 p;
      p.x = yb::pack_bf16x2(y.x, y.y);
      p.y = yb::pack_bf16x2(y.z, y.w);
      reinterpret_cast<uint2*>(reinterpret_cast<bf16*>(out) + static_cast<long long>(row) * ldo)[idx] = p;
    }
  }
}

template <int NV>
int launch_rmsnorm(const float* x, long long ldx, void* out, long long ldo, int out_f32, const float* w, int L, float eps,
                   cudaStream_t st) {
  const int blocks = (L + 7) / 8;
  if (out_f32)
    t5_rmsnorm_kernel<NV, true><<<blocks, 256, 0, st>>>(x, ldx, out, ldo, w, L, eps);
  else
    t5_rmsnorm_kernel<NV, false><<<blocks, 256, 0, st>>>(x, ldx, out, ldo, w, L, eps);
  return yb::check_launch("t5_rmsnorm");
}

// ------------------------------------------------------------------------------------------------
// gated GELU: out = bf16(u * gelu_tanh(g)), 8 columns per thread
// ------------------------------------------------------------------------------------------------
// the reference's GELU (wan/modules/t5.py:46-50) in fp32 with the accurate tanhf
__device__ __forceinline__ float t5_gelu(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;   // sqrt(2 / pi)
  return 0.5f * x * (1.0f + tanhf(k0 * (x + k1 * (x * x * x))));
}

__global__ void __launch_bounds__(256)
t5_geglu_kernel(const bf16* __restrict__ ug, long long ld, bf16* __restrict__ out, long long ldo, int L, int F) {
  const int chunks = F >> 3;
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= static_cast<long long>(L) * chunks) return;
  const long long row = idx / chunks;
  const int c = static_cast<int>(idx - row * chunks) * 8;
  const uint4 uu = *reinterpret_cast<const uint4*>(ug + row * ld + c);
  const uint4 gg = *reinterpret_cast<const uint4*>(ug + row * ld + F + c);
  const __nv_bfloat162* u2 = reinterpret_cast<const __nv_bfloat162*>(&uu);
  const __nv_bfloat162* g2 = reinterpret_cast<const __nv_bfloat162*>(&gg);
  uint32_t o[4];
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const float2 u = __bfloat1622float2(u2[p]);
    const float2 gv = __bfloat1622float2(g2[p]);
    o[p] = yb::pack_bf16x2(u.x * t5_gelu(gv.x), u.y * t5_gelu(gv.y));
  }
  *reinterpret_cast<uint4*>(out + row * ldo + c) = make_uint4(o[0], o[1], o[2], o[3]);
}

bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

}  // namespace

extern "C" int yb_t5_attention(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                               void* out, long long ldo, int B, int L, int heads, const void* bias, const void* key_mask,
                               void* stream) {
  if (!q || !k || !v || !out || !bias || B <= 0 || L <= 0 || heads <= 0) return YB_ERR_ARG;
  const long long W = static_cast<long long>(heads) * T5_HD;
  if (ldq < W || ldk < W || ldv < W || ldo < W || B > 65535 || heads > 65535 || L > (1 << 29)) return YB_ERR_SHAPE;
  if (misaligned16(q) || misaligned16(k) || misaligned16(v) || misaligned16(out) || (ldq | ldk | ldv | ldo) % 8)
    return YB_ERR_ALIGNMENT;
  const dim3 grid((L + T5_BQ - 1) / T5_BQ, heads, B);
  t5_attention_kernel<<<grid, T5_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      static_cast<const bf16*>(q), ldq, static_cast<const bf16*>(k), ldk, static_cast<const bf16*>(v), ldv,
      static_cast<bf16*>(out), ldo, L, static_cast<const float*>(bias), static_cast<const unsigned char*>(key_mask));
  return yb::check_launch("t5_attention");
}

extern "C" int yb_t5_rmsnorm(const void* x, long long ldx, void* out, long long ldo, int out_f32, const void* weight, int L,
                             int C, float eps, void* stream) {
  if (!x || !out || !weight || L <= 0 || C <= 0) return YB_ERR_ARG;
  if (ldx < C || ldo < C) return YB_ERR_SHAPE;
  if (misaligned16(x) || misaligned16(out) || misaligned16(weight) || ldx % 4 || ldo % (out_f32 ? 4 : 8))
    return YB_ERR_ALIGNMENT;
  const float* xf = static_cast<const float*>(x);
  const float* w = static_cast<const float*>(weight);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (C) {
    case 128: return launch_rmsnorm<1>(xf, ldx, out, ldo, out_f32, w, L, eps, st);
    case 256: return launch_rmsnorm<2>(xf, ldx, out, ldo, out_f32, w, L, eps, st);
    case 512: return launch_rmsnorm<4>(xf, ldx, out, ldo, out_f32, w, L, eps, st);
    case 768: return launch_rmsnorm<6>(xf, ldx, out, ldo, out_f32, w, L, eps, st);
    case 1024: return launch_rmsnorm<8>(xf, ldx, out, ldo, out_f32, w, L, eps, st);
    case 2048: return launch_rmsnorm<16>(xf, ldx, out, ldo, out_f32, w, L, eps, st);
    case 4096: return launch_rmsnorm<32>(xf, ldx, out, ldo, out_f32, w, L, eps, st);
    default: return YB_ERR_SHAPE;
  }
}

extern "C" int yb_t5_geglu(const void* ug, long long ld_ug, void* out, long long ldo, int L, int F, void* stream) {
  if (!ug || !out || L <= 0 || F <= 0) return YB_ERR_ARG;
  if (F % 8 || ld_ug < 2LL * F || ldo < F) return YB_ERR_SHAPE;
  if (misaligned16(ug) || misaligned16(out) || ld_ug % 8 || ldo % 8) return YB_ERR_ALIGNMENT;
  const long long n = static_cast<long long>(L) * (F / 8);
  const long long blocks = (n + 255) / 256;
  if (blocks > 0x7fffffffLL) return YB_ERR_SHAPE;
  t5_geglu_kernel<<<static_cast<unsigned>(blocks), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      static_cast<const bf16*>(ug), ld_ug, static_cast<bf16*>(out), ldo, L, F);
  return yb::check_launch("t5_geglu");
}
