// vae_elementwise.cu — the HBM-bound glue of the causal 3D VAE decoder (hyvideo/vae), channels-last bf16:
//   gn_stats          GroupNorm statistics (fp32 partials -> fp64 atomics)
//   pad_act           GroupNorm-apply + SiLU + nearest upsample + replicate padding in ONE gather pass that writes the
//                     padded input of the next implicit-GEMM conv (the reference runs GroupNorm, SiLU, interpolate,
//                     F.pad as four separate full-tensor passes: unet_causal_3d_blocks.py:72,144-174,375-379)
//   masked_softmax    frame-causal softmax of the mid-block attention scores (:37-45, diffusers Attention)
//   layout converters and the tile cross-fade (autoencoder_kl_causal_3d.py:343-359)
//   frame_match       the bitwise prefix / zero-tail scan of a resuming Wan VAE session (include/yume_b200_vae_resume.h)
#include "yb_host.h"
#include "../../include/yume_b200_stream.h"
#include "../../include/yume_b200_fp8_vae.h"
#include "../../include/yume_b200_vae_resume.h"
#include "../../include/yume_b200_vae_rows.h"
#include "../../include/yume_b200_vae_rows_enc.h"
#include "yb_ptx.cuh"

namespace yb {

// ---------------------------------------------------------------------------------------------------------
// GroupNorm statistics: x bf16 [N, C] (row stride ld) -> stats f64 [G][2] += (sum, sum of squares).
// Thread owns one 8-channel chunk and strides over voxels; per-channel fp32 partials (fixed order) -> fp64 atomics in smem per
// group -> fp64 global atomics: the only order-dependent sums are in double, so a decode is reproducible run to run (a float
// smem stage made statistics differ at 1e-7 between runs, enough to flip bf16 roundings that a deep decoder amplifies).
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gn_stats_kernel(const __nv_bfloat16* __restrict__ x, long long ld, double* __restrict__ stats, long long N, int C, int G) {
  __shared__ double sg[64][2];
  const int chunks = C >> 3;                 // 8-channel chunks per voxel
  const int vox_per_block = 256 / chunks;    // voxels handled per block iteration (chunks <= 256)
  const int tid = threadIdx.x;
  if (tid < 64) sg[tid][0] = sg[tid][1] = 0.0;
  __syncthreads();
  const int cg = C / G;                      // channels per group
  float s[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s[i] = q[i] = 0.f;
  if (tid < chunks * vox_per_block) {
    const int chunk = tid % chunks;
    for (long long v = static_cast<long long>(blockIdx.x) * vox_per_block + tid / chunks; v < N;
         v += static_cast<long long>(gridDim.x) * vox_per_block) {
      const uint4 raw = *reinterpret_cast<const uint4*>(x + v * ld + chunk * 8);
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = __bfloat1622float2(h[k]);
        s[2 * k] += f.x; q[2 * k] += f.x * f.x;
        s[2 * k + 1] += f.y; q[2 * k + 1] += f.y * f.y;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int g = (chunk * 8 + i) / cg;
      atomicAdd(&sg[g][0], static_cast<double>(s[i]));
      atomicAdd(&sg[g][1], static_cast<double>(q[i]));
    }
  }
  __syncthreads();
  if (tid < G) {
    atomicAdd(&stats[2 * tid], sg[tid][0]);
    atomicAdd(&stats[2 * tid + 1], sg[tid][1]);
  }
}

// ---------------------------------------------------------------------------------------------------------
// pad_act: out[tp,hp,wp,:] = act(gn(x[src(tp,hp,wp),:])), written to the replicate-padded (pad=1: [T+2,H+2,W+2,Cp]) or
// plain (pad=0: [T,H,W,Cp]) channels-last buffer. T,H,W are the OUTPUT dims (after the optional nearest upsample by
// (ft,fh,fw) of the source [Ts,Hs,Ws]); first frame is upsampled only spatially (UpsampleCausal3D, :156-163).
// Channels C..Cp-1 are written as zero.
// ---------------------------------------------------------------------------------------------------------
struct PadActParams {
  const __nv_bfloat16* x;
  long long ldx;
  __nv_bfloat16* out;
  const double* stats;   // null => no normalisation
  const float* gamma;
  const float* beta;
  int Ts, Hs, Ws, C, Cp, G;
  int T, H, W, ft, fh, fw;
  int pad, silu;
  float eps;
  double inv_count;      // 1 / (Ts*Hs*Ws*C/G)
};

__global__ void __launch_bounds__(256) pad_act_kernel(const PadActParams p) {
  // GroupNorm folded to one fma per element: y = x * a[c] + b[c], a = rstd_g * gamma, b = beta - mean_g * a, built once
  // per block in shared memory; all index math is 32-bit (the host rejects buffers with >= 2^31 16-byte chunks).
  __shared__ float s_a[1024], s_b[1024];
  const int chunks = p.Cp >> 3;
  const int Tp = p.T + 2 * p.pad, Hp = p.H + 2 * p.pad, Wp = p.W + 2 * p.pad;
  const int total = Tp * Hp * Wp * chunks;
  if (p.stats) {
    const int cg = p.C / p.G;
    for (int c = threadIdx.x; c < p.C; c += blockDim.x) {
      const int g = c / cg;
      const double mean = p.stats[2 * g] * p.inv_count;
      const double var = p.stats[2 * g + 1] * p.inv_count - mean * mean;
      const float a = rsqrtf(static_cast<float>(var) + p.eps) * __ldg(p.gamma + c);
      s_a[c] = a;
      s_b[c] = __ldg(p.beta + c) - static_cast<float>(mean) * a;
    }
    __syncthreads();
  }
  const bool plain = (p.stats == nullptr && !p.silu);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int chunk = i % chunks;
    int v = i / chunks;
    const int wp = v % Wp;
    v /= Wp;
    const int hp = v % Hp;
    const int tp = v / Hp;
    // output (unpadded) coordinate, clamped = replicate padding; temporal pad is 2 frames in FRONT only (causal)
    int t = p.pad ? max(tp - 2, 0) : tp;
    int h = p.pad ? min(max(hp - 1, 0), p.H - 1) : hp;
    int w = p.pad ? min(max(wp - 1, 0), p.W - 1) : wp;
    if (p.ft == 2) t = (t == 0) ? 0 : 1 + ((t - 1) >> 1);
    if (p.fh == 2) h >>= 1; else h /= p.fh;
    if (p.fw == 2) w >>= 1; else w /= p.fw;
    uint4 o = make_uint4(0u, 0u, 0u, 0u);
    const int c0 = chunk * 8;
    if (c0 < p.C) {
      const long long src = (static_cast<long long>(t) * p.Hs + h) * p.Ws + w;
      const uint4 raw = *reinterpret_cast<const uint4*>(p.x + src * p.ldx + c0);
      if (plain) {
        o = raw;
      } else {
        const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&raw);
        float f[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 t2 = __bfloat1622float2(hh[k]);
          f[2 * k] = t2.x;
          f[2 * k + 1] = t2.y;
        }
        if (p.stats) {
#pragma unroll
          for (int k = 0; k < 8; ++k) f[k] = fmaf(f[k], s_a[c0 + k], s_b[c0 + k]);
        }
        if (p.silu) {
#pragma unroll
          for (int k = 0; k < 8; ++k) f[k] = f[k] / (1.f + __expf(-f[k]));
        }
        o = make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
      }
    }
    *reinterpret_cast<uint4*>(p.out + static_cast<long long>(i) * 8) = o;
  }
}

// frame-causal softmax: S f32 [L, ldS] -> P bf16 [L, ldP]; row i keeps keys j < (i / hw + 1) * hw, others become 0
__global__ void __launch_bounds__(256)
masked_softmax_kernel(const float* __restrict__ S, long long ldS, __nv_bfloat16* __restrict__ P, long long ldP, int L,
                      int hw) {
  __shared__ float red[8];
  const int row = blockIdx.x;
  const int nvalid = min(L, (row / hw + 1) * hw);
  const float* s = S + static_cast<long long>(row) * ldS;
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < nvalid; j += 256) mx = fmaxf(mx, s[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int j = threadIdx.x; j < nvalid; j += 256) sum += __expf(s[j] - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) sum += red[i];
  const float inv = 1.f / sum;
  __nv_bfloat16* pr = P + static_cast<long long>(row) * ldP;
  for (int j = threadIdx.x; j < ldP; j += 256)
    pr[j] = __float2bfloat16_rn(j < nvalid ? __expf(s[j] - mx) * inv : 0.f);
}

// z f32 [Cn, N] (NCDHW, N = T*H*W; channel planes `plane` elements apart) -> bf16 [N, ldo] channels-last, columns >= Cn zero
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out, long long N, int Cn,
                                    int ldo, long long plane) {
  const long long total = N * ldo;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % ldo);
    const long long v = i / ldo;
    out[i] = __float2bfloat16_rn(c < Cn ? x[static_cast<long long>(c) * plane + v] : 0.f);
  }
}

// x f32 [N, ldx] channels-last -> out f32 [Cn, N], channel planes `plane` elements apart (N for a dense result)
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ x, long long ldx, float* __restrict__ out, long long N,
                                    int Cn, float lo, float hi, long long plane) {
  const long long total = N * Cn;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long v = i % N;
    const int c = static_cast<int>(i / N);
    out[c * plane + v] = fminf(fmaxf(x[v * ldx + c], lo), hi);
  }
}

// One cross-fade step of blend_v / blend_h / blend_t: `a * (1 - y / ext) + b * (y / ext)` on f32 tensors. Python computes both
// weights in double and torch rounds them to f32; each product and the sum is rounded on its own (no fused multiply-add).
__device__ __forceinline__ float xfade(float a, float b, int y, int ext) {
  const double r = static_cast<double>(y) / static_cast<double>(ext);
  return __fadd_rn(__fmul_rn(a, static_cast<float>(1.0 - r)), __fmul_rn(b, static_cast<float>(r)));
}

// cross-fade along one axis of contiguous f32 [C, T, H, W] tiles (blend_v / blend_h / blend_t):
//   b[.., y, ..] = a[.., ea - ext + y, ..] * (1 - y/ext) + b[.., y, ..] * (y/ext)   for y < ext   (xfade: the reference's roundings)
// a has extent `ea` on the blend axis, b has `eb`; all other extents equal. outer/inner: product of the dims before /
// after the axis.
__global__ void blend_kernel(const float* __restrict__ a, float* __restrict__ b, long long outer, int ea, int eb, int ext,
                             long long inner, long long a_outer_stride, long long b_outer_stride) {
  const long long total = outer * ext * inner;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long in = i % inner;
    const int y = static_cast<int>((i / inner) % ext);
    const long long o = i / (inner * ext);
    const float av = a[o * a_outer_stride + static_cast<long long>(ea - ext + y) * inner + in];
    float* bp = b + o * b_outer_stride + static_cast<long long>(y) * inner + in;
    *bp = xfade(av, *bp, y, ext);
  }
}

// ---------------------------------------------------------------------------------------------------------
// One-pass assembly of a tiled decode (AutoencoderKLCausal3D.temporal_tiled_decode / spatial_tiled_decode,
// hyvideo/vae/autoencoder_kl_causal_3d.py:417-463, 500-531). The reference decodes tile after tile, cross-fades each tile IN PLACE
// with its upper / left / previous neighbour (blend_v, blend_h, blend_t, :343-359), crops and torch.cat's rows, then columns, then
// time. Every output voxel is therefore a fixed expression of at most 2 (time) x 4 (space) RAW tile values; this kernel evaluates
// that expression directly from the raw tiles into the final [C, F, H, W] video — same operations, same order, same fp32
// roundings as the in-place sequence (xfade below), bit for bit — so tiles can be decoded in any order, on any GPU.
// A neighbour enters with its own blends applied only where they touch the rows / columns / frames read from it, which holds
// when no tile is read back inside its own blended region: size(k) >= ext(k) + ext(k+1) for every interior tile k
// (ops.vae_assemble_tiles checks it; tile overlap factors <= 0.5 always satisfy it).
//   tiles   table of raw decoded tiles: tile (ti, i, j) is f32 [C, ft, h_i, w_j] contiguous at ptr[(ti*ni + i)*nj + j]
//   space   tile (i, j) covers output rows [i*rl, i*rl + min(rl, h_i)), blended over its first ev rows with tile (i-1, j):
//           ev = min(h_{i-1}, h_i, E) (blend_v clamps the extent to both tiles); columns likewise
//   time    temporal tile ti (its first decoded frame already dropped for ti > 0) covers frames [f0(ti), f0(ti) + keep(ti)),
//           blended over its first min(len_{ti-1}, len_ti, Et) frames with the last frames of tile ti-1
// ---------------------------------------------------------------------------------------------------------
struct TileAsm {
  const float* const* ptr;   // [nt * ni * nj] device pointers
  const int* th;             // [ni] tile heights (output pixels)
  const int* tw;             // [nj] tile widths
  const int* tlen;           // [nt] frames per temporal tile (after the drop)
  const int* tf0;            // [nt] first output frame of temporal tile ti
  int nt, ni, nj, C, F, H, W;
  int rl, E;                 // spatial row_limit / blend extent (0 = untiled in space: ni == nj == 1)
  int tl, Et;                // temporal keep limit / blend extent
};

__device__ __forceinline__ float tile_at(const TileAsm& a, int ti, int i, int j, int c, int f, int y, int x) {
  const float* t = a.ptr[(ti * a.ni + i) * a.nj + j];
  const int skip = ti > 0 ? 1 : 0;   // later temporal tiles: the first decoded frame is dropped (dec[:, :, 1:], :519-520)
  return t[((static_cast<long long>(c) * (a.tlen[ti] + skip) + f + skip) * a.th[i] + y) * a.tw[j] + x];
}
// fully blended value of spatial tile (i, j) of temporal tile ti at (y, x): blend_v with the upper neighbour first, then blend_h
// with the left neighbour (the reference's order, :440-448); neighbours enter with THEIR blends applied, which for the rows /
// columns read here (their last `ext` ones) reduces to one more blend with raw tiles
__device__ __forceinline__ float spatial_value(const TileAsm& a, int ti, int i, int j, int c, int f, int y, int x) {
  const int ev = i > 0 ? min(min(a.th[i - 1], a.th[i]), a.E) : 0;
  const int eh = j > 0 ? min(min(a.tw[j - 1], a.tw[j]), a.E) : 0;
  const bool bv = y < ev, bh = x < eh;
  float v = tile_at(a, ti, i, j, c, f, y, x);
  if (bv) {   // upper tile's row (already blended horizontally with ITS left neighbour on these columns)
    const int r = a.th[i - 1] - ev + y;
    float u = tile_at(a, ti, i - 1, j, c, f, r, x);
    if (bh) u = xfade(tile_at(a, ti, i - 1, j - 1, c, f, r, a.tw[j - 1] - eh + x), u, x, eh);
    v = xfade(u, v, y, ev);
  }
  if (bh) {   // left tile's column (already blended vertically with ITS upper neighbour on these rows)
    const int cx = a.tw[j - 1] - eh + x;
    float lft = tile_at(a, ti, i, j - 1, c, f, y, cx);
    if (bv) lft = xfade(tile_at(a, ti, i - 1, j - 1, c, f, a.th[i - 1] - ev + y, cx), lft, y, ev);
    v = xfade(lft, v, x, eh);
  }
  return v;
}

__global__ void __launch_bounds__(256) vae_assemble_tiles_kernel(const TileAsm a, float* __restrict__ out) {
  const long long total = static_cast<long long>(a.C) * a.F * a.H * a.W;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int X = static_cast<int>(idx % a.W);
    const int Y = static_cast<int>((idx / a.W) % a.H);
    const int Fo = static_cast<int>((idx / (static_cast<long long>(a.W) * a.H)) % a.F);
    const int c = static_cast<int>(idx / (static_cast<long long>(a.W) * a.H * a.F));
    int i = 0, y = Y, j = 0, x = X;
    if (a.rl > 0) {
      i = min(Y / a.rl, a.ni - 1); y = Y - i * a.rl;
      j = min(X / a.rl, a.nj - 1); x = X - j * a.rl;
    }
    int ti = a.nt - 1;
    while (ti > 0 && Fo < a.tf0[ti]) --ti;
    const int f = Fo - a.tf0[ti];
    float v = spatial_value(a, ti, i, j, c, f, y, x);
    if (ti > 0) {
      const int et = min(min(a.tlen[ti - 1], a.tlen[ti]), a.Et);
      if (f < et) v = xfade(spatial_value(a, ti - 1, i, j, c, a.tlen[ti - 1] - et + f, y, x), v, f, et);
    }
    out[idx] = v;
  }
}

// ---------------------------------------------------------------------------------------------------------
// Wan2.2 VAE glue (wan23/modules/vae2_2.py).
// rms_act: one warp per OUTPUT voxel: [RMS_norm over channels (F.normalize * sqrt(C) * gamma, :47-61)] -> [SiLU] ->
// nearest-exact 2x spatial upsample (:64-70, Resample :95-101), written channels-last [T, H*f, W*f, Cp] (no padding:
// the conv takes its zero padding from TMA out-of-bounds fill).
// ---------------------------------------------------------------------------------------------------------
// NCH = 16-byte chunks per lane per voxel, G = lanes per voxel (G < 32 only with NCH == 1: narrow rows share a warp).
// A warp keeps U * (32 / G) voxels in flight, U = 4 / NCH. All index math is 32-bit and the f == 1 path has none.
// BAND (yb_vae_rms_act_rows): out is a band buffer [T, H + 2, W, Cp] written at rows 1 .. H, and the first and last written row of
// every frame also go to send [2, T, W, Cp] when it is not NULL; the values are those of the dense form.
template <int NCH, int G, bool BAND = false>
__global__ void __launch_bounds__(256)
rms_act_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ out, const float* __restrict__ gamma,
               int T, int Hs, int Ws, int C, int Cp, int f, int silu, __nv_bfloat16* __restrict__ send = nullptr) {
  constexpr int U = 4 / NCH;
  constexpr int SUB = 32 / G;                     // voxels side by side in one warp
  constexpr int VPI = U * SUB;                    // voxels per warp iteration
  const int H = Hs * f, W = Ws * f;
  const int nvox = T * H * W;
  const int lane = threadIdx.x & 31;
  const int gl = lane % G, sub = lane / G;
  const int cch = C >> 3, pch = Cp >> 3;
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
      const int v = v0 + u * SUB + sub;
      if (v >= nvox) continue;
      const float sc = gamma ? sqrt_c / fmaxf(sqrtf(scl[u]), 1e-12f) : 1.f;
#pragma unroll
      for (int j = 0; j < NCH; ++j) {
        const int c = gl + G * j;
        if (c >= pch) continue;
        uint4 o = make_uint4(0u, 0u, 0u, 0u);
        if (c < cch) {
          const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&raw[u][j]);
          float y[8];
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
          o = make_uint4(pack_bf16x2(y[0], y[1]), pack_bf16x2(y[2], y[3]), pack_bf16x2(y[4], y[5]), pack_bf16x2(y[6], y[7]));
        }
        if constexpr (BAND) {
          const int w = v % W, r = v / W;
          const int h = r % H, t = r / H;
          *reinterpret_cast<uint4*>(out + (static_cast<long long>(t * (H + 2) + h + 1) * W + w) * Cp + c * 8) = o;
          if (send) {
            if (h == 0) *reinterpret_cast<uint4*>(send + (static_cast<long long>(t) * W + w) * Cp + c * 8) = o;
            if (h == H - 1) *reinterpret_cast<uint4*>(send + (static_cast<long long>(T + t) * W + w) * Cp + c * 8) = o;
          }
        } else {
          *reinterpret_cast<uint4*>(out + static_cast<long long>(v) * Cp + c * 8) = o;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// RMS_norm (* gamma) -> SiLU -> nearest 2x upsample -> bf16 rounding -> 1x128 e4m3 quantisation per voxel.
// Lane layout and fp32 arithmetic are those of rms_act_kernel<NCH, G> above for the same C / Cp, so the bf16 values
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
        group_scale(amax, inv, scale);
        *reinterpret_cast<uint2*>(out + static_cast<long long>(v) * Cp + c * 8) =
            make_uint2(cvt_e4m3x4(y[0] * inv, y[1] * inv, y[2] * inv, y[3] * inv),
                       cvt_e4m3x4(y[4] * inv, y[5] * inv, y[6] * inv, y[7] * inv));
        if ((c & 15) == 0) {
          const int t = v / HW;
          out_scale[(static_cast<long long>(t) * groups + (c >> 4)) * HW + (v - t * HW)] = scale;
        }
      }
    }
  }
}

// main[f', h', w', oc] += x[t, h, w, ci]: the DupUp3D shortcut (:376-418) of Up_ResidualBlock (:499-503) on the whole
// sequence, first `drop` duplicated frames dropped (ft-1 on the first chunk of a sequence, 0 on the chunks after it).
// d = f' + drop, t = d / ft, a = d % ft, e = ((oc*ft + a)*fs + b)*fs + c, ci = e / rep with rep = out_c*ft*fs*fs / in_c.
__global__ void __launch_bounds__(256)
dupup_add_kernel(__nv_bfloat16* __restrict__ main_, const __nv_bfloat16* __restrict__ x, int Ts, int Hs, int Ws, int in_c,
                 int out_c, int ft, int fs, int drop) {
  // one thread = 8 consecutive output channels of one output voxel: a 16-byte read-modify-write of main, eight gathers
  // from the (8x..16x smaller, cache-resident) source voxel
  const int To = ft * Ts - drop, Ho = Hs * fs, Wo = Ws * fs;
  const int rep = out_c * ft * fs * fs / in_c;
  const int rsh = (rep & (rep - 1)) == 0 ? 31 - __clz(rep) : -1;   // rep is 2, 4 or 8 in both Wan VAEs: shift, no division
  const int chunks = out_c >> 3;
  const int estep = ft * fs * fs;
  const long long total = static_cast<long long>(To) * Ho * Wo * chunks;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i / chunks);
    const int oc = static_cast<int>(i - static_cast<long long>(v) * chunks) << 3;
    const int wo = v % Wo;
    const int r = v / Wo;
    const int ho = r % Ho;
    const int fo = r / Ho;
    const int d = fo + drop;
    const int t = d / ft, a = d % ft;
    const int e0 = ((oc * ft + a) * fs + (ho % fs)) * fs + (wo % fs);
    const __nv_bfloat16* xs = x + ((static_cast<long long>(t) * Hs + ho / fs) * Ws + wo / fs) * in_c;
    uint4* mp = reinterpret_cast<uint4*>(main_ + static_cast<long long>(v) * out_c + oc);
    uint4 raw = *mp;
    __nv_bfloat162* hh = reinterpret_cast<__nv_bfloat162*>(&raw);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 m = __bfloat1622float2(hh[k]);
      const int ea = e0 + (2 * k) * estep, eb = ea + estep;
      const float a0 = __bfloat162float(xs[rsh >= 0 ? (ea >> rsh) : ea / rep]);
      const float a1 = __bfloat162float(xs[rsh >= 0 ? (eb >> rsh) : eb / rep]);
      hh[k] = __floats2bfloat162_rn(m.x + a0, m.y + a1);
    }
    *mp = raw;
  }
}

// AvgDown3D shortcut of the Wan2.2 encoder's Down_ResidualBlock (vae2_2.py:320-373, 449-459) over the whole frame sequence:
// pad_t = (ft - T % ft) % ft zero frames in FRONT, 'b c (t a) (h q) (w r) -> b (c a q r) t h w', then the mean over groups of
// G = in_c*ft*fs*fs / out_c consecutive channels. main[to, ho, wo, oc] += mean_g x[c, to*ft + a - pad_t, ho*fs + q, wo*fs + r]
// with ((c*ft + a)*fs + q)*fs + r = oc*G + g. One thread = 8 consecutive output channels of one output voxel.
__global__ void __launch_bounds__(256)
avgdown_add_kernel(__nv_bfloat16* __restrict__ main_, const __nv_bfloat16* __restrict__ x, int T, int H, int W, int in_c,
                   int out_c, int ft, int fs) {
  const int pad_t = (ft - T % ft) % ft;
  const int To = (T + pad_t) / ft, Ho = H / fs, Wo = W / fs;
  const int G = in_c * ft * fs * fs / out_c, per_c = ft * fs * fs;
  const int chunks = out_c >> 3;
  const float inv = 1.0f / static_cast<float>(G);
  const long long total = static_cast<long long>(To) * Ho * Wo * chunks;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i / chunks);
    const int oc = static_cast<int>(i - static_cast<long long>(v) * chunks) << 3;
    const int wo = v % Wo;
    const int rr = v / Wo;
    const int ho = rr % Ho;
    const int to = rr / Ho;
    uint4* mp = reinterpret_cast<uint4*>(main_ + static_cast<long long>(v) * out_c + oc);
    uint4 raw = *mp;
    __nv_bfloat16* hh = reinterpret_cast<__nv_bfloat16*>(&raw);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float acc = 0.0f;
      for (int g = 0; g < G; ++g) {
        const int j = (oc + k) * G + g;
        const int c = j / per_c, rem = j - c * per_c;
        const int a = rem / (fs * fs), q = (rem / fs) % fs, r = rem % fs;
        const int ti = to * ft + a - pad_t;
        if (ti >= 0)
          acc += __bfloat162float(x[((static_cast<long long>(ti) * H + ho * fs + q) * W + wo * fs + r) * in_c + c]);
      }
      hh[k] = __float2bfloat16_rn(__bfloat162float(hh[k]) + acc * inv);
    }
    *mp = raw;
  }
}

// video f32 [3, T, H, W] -> out bf16 [T*(H/2)*(W/2), ldo], channel (c r q) = c*4 + r*2 + q <- video[c, f, 2h + q, 2w + r]
// (patchify 'b c f (h q) (w r) -> b (c r q) f h w', vae2_2.py:284-300); columns 12..ldo-1 are zeroed (TMA reads 64-channel chunks)
__global__ void patchify2_bf16_kernel(const float* __restrict__ video, __nv_bfloat16* __restrict__ out, long long ldo, int T,
                                      int H, int W, long long plane) {
  const int Hh = H / 2, Wh = W / 2;
  const long long total = static_cast<long long>(T) * Hh * Wh;
  for (long long v = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; v < total;
       v += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int w = static_cast<int>(v % Wh);
    const long long rr = v / Wh;
    const int h = static_cast<int>(rr % Hh);
    const int f = static_cast<int>(rr / Hh);
    __nv_bfloat16* o = out + v * ldo;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* src = video + c * plane + (static_cast<long long>(f) * H + 2 * h) * W + 2 * w;
      const float2 top = *reinterpret_cast<const float2*>(src);          // q = 0: r = 0, 1
      const float2 bot = *reinterpret_cast<const float2*>(src + W);      // q = 1
      o[c * 4 + 0] = __float2bfloat16_rn(top.x);   // r = 0, q = 0
      o[c * 4 + 1] = __float2bfloat16_rn(bot.x);   // r = 0, q = 1
      o[c * 4 + 2] = __float2bfloat16_rn(top.y);   // r = 1, q = 0
      o[c * 4 + 3] = __float2bfloat16_rn(bot.y);   // r = 1, q = 1
    }
    for (int c = 12; c < ldo; ++c) o[c] = __float2bfloat16_rn(0.0f);
  }
}

// y f32 [T*H*W, ldy] (12 valid channels) -> out f32 [3, T, 2H, 2W], clamp to [-1, 1]:
// unpatchify 'b (c r q) f h w -> b c f (h q) (w r)' (:305-319) + Wan2_2_VAE.decode's clamp_ (:1066-1067)
__global__ void unpatchify2_clamp_kernel(const float* __restrict__ y, long long ldy, float* __restrict__ out, int T, int H,
                                         int W, long long plane) {
  const long long total = 3LL * T * (2 * H) * (2 * W);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int wo = static_cast<int>(i % (2 * W));
    long long v = i / (2 * W);
    const int ho = static_cast<int>(v % (2 * H));
    v /= (2 * H);
    const int f = static_cast<int>(v % T);
    const int c = static_cast<int>(v / T);
    const int q = ho & 1, r = wo & 1;
    const float val = y[((static_cast<long long>(f) * H + (ho >> 1)) * W + (wo >> 1)) * ldy + (c * 2 + r) * 2 + q];
    out[c * plane + (i - static_cast<long long>(c) * T * (2 * H) * (2 * W))] = fminf(fmaxf(val, -1.f), 1.f);
  }
}

// Row-band form of unpatchify2_clamp_kernel (include/yume_b200_vae_rows.h): the band's 2Hs rows of T frames, frames `frame`
// elements apart, rows 2W apart
__global__ void unpatchify2_clamp_rows_kernel(const float* __restrict__ y, long long ldy, float* __restrict__ out, int T, int Hs,
                                              int W, long long plane, long long frame) {
  const long long total = 3LL * T * (2 * Hs) * (2 * W);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int wo = static_cast<int>(i % (2 * W));
    long long v = i / (2 * W);
    const int ho = static_cast<int>(v % (2 * Hs));
    v /= (2 * Hs);
    const int f = static_cast<int>(v % T);
    const int c = static_cast<int>(v / T);
    const int q = ho & 1, r = wo & 1;
    const float val = y[((static_cast<long long>(f) * Hs + (ho >> 1)) * W + (wo >> 1)) * ldy + (c * 2 + r) * 2 + q];
    out[c * plane + f * frame + static_cast<long long>(ho) * (2 * W) + wo] = fminf(fmaxf(val, -1.f), 1.f);
  }
}

// Row-band form of nhwc_to_nchw_kernel: x f32 [T*Hs*W, ldx] -> Cn channels x T frames (`frame` apart) x Hs rows x W columns
__global__ void nhwc_to_nchw_rows_kernel(const float* __restrict__ x, long long ldx, float* __restrict__ out, int T, int Hs, int W,
                                         int Cn, float lo, float hi, long long plane, long long frame) {
  const long long N = static_cast<long long>(T) * Hs * W;
  const long long total = N * Cn;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long v = i % N;
    const int c = static_cast<int>(i / N);
    const long long f = v / (static_cast<long long>(Hs) * W), hw = v % (static_cast<long long>(Hs) * W);
    out[c * plane + f * frame + hw] = fminf(fmaxf(x[v * ldx + c], lo), hi);
  }
}

// Halo glue of a band buffer [T, Hs + 2, nvec] (16-byte words): pack copies rows 1 and Hs into send [2, T, nvec]; unpack copies
// recv_top / recv_bot [T, nvec] into rows 0 and Hs + 1, zeros for a NULL source
__global__ void rows_pack_kernel(const uint4* __restrict__ buf, uint4* __restrict__ send, int T, int Hs, long long nvec) {
  const long long total = 2LL * T * nvec;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long e = i % nvec, r = i / nvec;
    const int t = static_cast<int>(r % T), side = static_cast<int>(r / T);
    send[i] = buf[(static_cast<long long>(t) * (Hs + 2) + (side ? Hs : 1)) * nvec + e];
  }
}

__global__ void rows_unpack_kernel(const uint4* __restrict__ top, const uint4* __restrict__ bot, uint4* __restrict__ buf, int T,
                                   int Hs, long long nvec) {
  const long long total = 2LL * T * nvec;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long e = i % nvec, r = i / nvec;
    const int t = static_cast<int>(r % T), side = static_cast<int>(r / T);
    const uint4* src = side ? bot : top;
    buf[(static_cast<long long>(t) * (Hs + 2) + (side ? Hs + 1 : 0)) * nvec + e] =
        src ? src[static_cast<long long>(t) * nvec + e] : make_uint4(0u, 0u, 0u, 0u);
  }
}

// Band readers of a row-parallel encode (include/yume_b200_vae_rows_enc.h): the T frames of a band buffer [T, hs + 2, Wo, ldo],
// buffer row j = image row r0 - 1 + j of the level (zeros outside the image), each element converted as the _win readers do
__global__ void patchify2_bf16_rows_kernel(const float* __restrict__ video, __nv_bfloat16* __restrict__ out, int ldo, int T,
                                           int H, int W, long long plane, int r0, int hs) {
  const int Hh = H / 2, Wh = W / 2;
  const long long total = static_cast<long long>(T) * (hs + 2) * Wh;
  for (long long v = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; v < total;
       v += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int w = static_cast<int>(v % Wh);
    const long long rr = v / Wh;
    const int h = r0 - 1 + static_cast<int>(rr % (hs + 2));
    const int f = static_cast<int>(rr / (hs + 2));
    __nv_bfloat16* o = out + v * ldo;
    int c0 = 0;
    if (h >= 0 && h < Hh) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float* src = video + c * plane + (static_cast<long long>(f) * H + 2 * h) * W + 2 * w;
        const float2 top = *reinterpret_cast<const float2*>(src);
        const float2 bot = *reinterpret_cast<const float2*>(src + W);
        o[c * 4 + 0] = __float2bfloat16_rn(top.x);
        o[c * 4 + 1] = __float2bfloat16_rn(bot.x);
        o[c * 4 + 2] = __float2bfloat16_rn(top.y);
        o[c * 4 + 3] = __float2bfloat16_rn(bot.y);
      }
      c0 = 12;
    }
    for (int c = c0; c < ldo; ++c) o[c] = __float2bfloat16_rn(0.0f);
  }
}

__global__ void nchw_to_nhwc_rows_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out, int ldo, int T, int H,
                                         int W, int Cn, long long plane, int r0, int hs) {
  const long long total = static_cast<long long>(T) * (hs + 2) * W * ldo;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % ldo);
    const long long v = i / ldo;
    const int w = static_cast<int>(v % W);
    const long long rr = v / W;
    const int h = r0 - 1 + static_cast<int>(rr % (hs + 2));
    const int f = static_cast<int>(rr / (hs + 2));
    out[i] = __float2bfloat16_rn(c < Cn && h >= 0 && h < H ? x[static_cast<long long>(c) * plane + (static_cast<long long>(f) * H + h) * W + w]
                                                            : 0.f);
  }
}

inline int grid_for(long long total) {
  long long b = (total + 255) / 256;
  const long long cap = static_cast<long long>(sm_count()) * 16;
  return static_cast<int>(b < cap ? (b > 0 ? b : 1) : cap);
}

// ---------------------------------------------------------------------------------------------------------
// Frame comparison of a resuming VAE session (include/yume_b200_vae_resume.h). kept [C, t_kept, nvec] and x [C, t, nvec] in
// V-sized words. A work item is FM_VEC_PER_THREAD * 256 words of one (channel, frame) row: its threads OR together x's bits
// and the XOR of x with kept, the block ORs the two flags, and thread 0 lowers result[0] to the frame on a difference and
// raises result[1] past the frame on a set bit. Only the atomics depend on the order of blocks, and min / max do not.
// ---------------------------------------------------------------------------------------------------------
constexpr int FM_VEC_PER_THREAD = 8;

__device__ __forceinline__ unsigned long long fm_bits(uint4 v) {
  return static_cast<unsigned long long>(v.x | v.y) | (static_cast<unsigned long long>(v.z | v.w) << 32);
}
__device__ __forceinline__ uint4 fm_xor(uint4 a, uint4 b) { return make_uint4(a.x ^ b.x, a.y ^ b.y, a.z ^ b.z, a.w ^ b.w); }
template <typename V> __device__ __forceinline__ unsigned long long fm_bits(V v) { return static_cast<unsigned long long>(v); }
template <typename V> __device__ __forceinline__ V fm_xor(V a, V b) { return static_cast<V>(a ^ b); }

__global__ void frame_match_init_kernel(int* result, int n_cmp) {
  result[0] = n_cmp;
  result[1] = 0;
}

template <typename V>
__global__ void __launch_bounds__(256) frame_match_kernel(const V* __restrict__ kept, int t_kept, const V* __restrict__ x, int t,
                                                          long long rows, long long nvec, int* __restrict__ result) {
  const long long per_item = static_cast<long long>(FM_VEC_PER_THREAD) * blockDim.x;
  const long long items_per_row = (nvec + per_item - 1) / per_item;
  for (long long item = blockIdx.x; item < rows * items_per_row; item += gridDim.x) {
    const long long row = item / items_per_row;
    const long long base = (item % items_per_row) * per_item;
    const int f = static_cast<int>(row % t);
    const long long c = row / t;
    const V* xr = x + row * nvec;
    const V* kr = f < t_kept ? kept + (c * t_kept + f) * nvec : nullptr;
    unsigned long long nz = 0, diff = 0;
#pragma unroll
    for (int j = 0; j < FM_VEC_PER_THREAD; ++j) {
      const long long i = base + static_cast<long long>(j) * blockDim.x + threadIdx.x;
      if (i < nvec) {
        const V a = xr[i];
        nz |= fm_bits(a);
        if (kr) diff |= fm_bits(fm_xor(a, kr[i]));
      }
    }
    const int any_nz = __syncthreads_or(nz != 0);
    const int any_diff = __syncthreads_or(diff != 0);
    if (threadIdx.x == 0) {
      if (any_diff) atomicMin(result, f);
      if (any_nz) atomicMax(result + 1, f + 1);
    }
  }
}

}  // namespace yb

using namespace yb;

extern "C" int yb_gn_stats(const void* x, long long ld, void* stats, long long N, int C, int G, void* stream_) {
  if (!x || !stats || N <= 0 || C <= 0 || G <= 0) return YB_ERR_ARG;
  if (C % 8 != 0 || C % G != 0 || C > 2048 || G > 64) return YB_ERR_SHAPE;
  if ((ld % 8) || (reinterpret_cast<uintptr_t>(x) & 0xF)) return YB_ERR_ALIGNMENT;
  const int vox_per_block = 256 / (C / 8);
  long long blocks = (N + vox_per_block - 1) / vox_per_block;
  if (blocks > sm_count() * 8) blocks = sm_count() * 8;
  gn_stats_kernel<<<static_cast<int>(blocks), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __nv_bfloat16*>(x), ld, static_cast<double*>(stats), N, C, G);
  return check_launch("gn_stats");
}

extern "C" int yb_vae_pad_act(const void* x, long long ldx, int Ts, int Hs, int Ws, int C, void* out, int Cp, int pad,
                              int ft, int fh, int fw, const void* stats, const void* gamma, const void* beta, int G,
                              float eps, int silu, void* stream_) {
  if (!x || !out || Ts <= 0 || Hs <= 0 || Ws <= 0 || C <= 0) return YB_ERR_ARG;
  if (C % 8 != 0 || Cp % 8 != 0 || Cp < C || (ft != 1 && ft != 2) || fh < 1 || fw < 1) return YB_ERR_SHAPE;
  if (stats && (!gamma || !beta || G <= 0 || C % G != 0)) return YB_ERR_ARG;
  if ((ldx % 8) || (reinterpret_cast<uintptr_t>(x) & 0xF) || (reinterpret_cast<uintptr_t>(out) & 0xF)) return YB_ERR_ALIGNMENT;
  PadActParams p;
  p.x = static_cast<const __nv_bfloat16*>(x);
  p.ldx = ldx;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.stats = static_cast<const double*>(stats);
  p.gamma = static_cast<const float*>(gamma);
  p.beta = static_cast<const float*>(beta);
  p.Ts = Ts; p.Hs = Hs; p.Ws = Ws; p.C = C; p.Cp = Cp; p.G = G;
  p.T = (ft == 2) ? 1 + 2 * (Ts - 1) : Ts;
  p.H = Hs * fh; p.W = Ws * fw;
  p.ft = ft; p.fh = fh; p.fw = fw;
  p.pad = pad ? 1 : 0; p.silu = silu;
  p.eps = eps;
  p.inv_count = stats ? 1.0 / (static_cast<double>(Ts) * Hs * Ws * (C / G)) : 0.0;
  const long long total = static_cast<long long>(p.T + 2 * p.pad) * (p.H + 2 * p.pad) * (p.W + 2 * p.pad) * (Cp / 8);
  if (total > 0x7fffffffLL - (1LL << 26) || (stats && C > 1024)) return YB_ERR_SHAPE;   // 32-bit indices, smem scale table
  pad_act_kernel<<<grid_for(total), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
  return check_launch("vae_pad_act");
}

extern "C" int yb_masked_softmax(const void* S, long long ldS, void* P, long long ldP, int L, int hw, void* stream_) {
  if (!S || !P || L <= 0 || hw <= 0 || ldP < L || ldS < L) return YB_ERR_ARG;
  masked_softmax_kernel<<<L, 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(S), ldS, static_cast<__nv_bfloat16*>(P), ldP, L, hw);
  return check_launch("masked_softmax");
}

extern "C" int yb_nchw_to_nhwc_bf16_win(const void* x, long long plane, void* out, long long N, int Cn, int ldo, void* stream_) {
  if (!x || !out || N <= 0 || Cn <= 0 || ldo < Cn || plane < N) return YB_ERR_ARG;
  nchw_to_nhwc_kernel<<<grid_for(N * ldo), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(x), static_cast<__nv_bfloat16*>(out), N, Cn, ldo, plane);
  return check_launch("nchw_to_nhwc");
}

extern "C" int yb_nchw_to_nhwc_bf16(const void* x, void* out, long long N, int Cn, int ldo, void* stream_) {
  return yb_nchw_to_nhwc_bf16_win(x, N, out, N, Cn, ldo, stream_);
}

extern "C" int yb_nhwc_to_nchw_f32(const void* x, long long ldx, void* out, long long N, int Cn, void* stream_) {
  if (!x || !out || N <= 0 || Cn <= 0 || ldx < Cn) return YB_ERR_ARG;
  nhwc_to_nchw_kernel<<<grid_for(N * Cn), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(x), ldx, static_cast<float*>(out), N, Cn, -INFINITY, INFINITY, N);
  return check_launch("nhwc_to_nchw");
}

extern "C" int yb_nhwc_to_nchw_f32_clamp(const void* x, long long ldx, void* out, long long N, int Cn, float lo, float hi,
                                         void* stream_) {
  if (!x || !out || N <= 0 || Cn <= 0 || ldx < Cn || !(lo <= hi)) return YB_ERR_ARG;
  nhwc_to_nchw_kernel<<<grid_for(N * Cn), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(x), ldx, static_cast<float*>(out), N, Cn, lo, hi, N);
  return check_launch("nhwc_to_nchw_clamp");
}

extern "C" int yb_blend(const void* a, void* b, long long outer, int ea, int eb, int ext, long long inner,
                        void* stream_) {
  if (!a || !b || outer <= 0 || ext <= 0 || inner <= 0 || ext > ea || ext > eb) return YB_ERR_ARG;
  blend_kernel<<<grid_for(outer * ext * inner), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(a), static_cast<float*>(b), outer, ea, eb, ext, inner,
      static_cast<long long>(ea) * inner, static_cast<long long>(eb) * inner);
  return check_launch("blend");
}


extern "C" int yb_vae_assemble_tiles(const void* const* tile_ptrs, const int* th, const int* tw, const int* tlen, const int* tf0,
                                     int nt, int ni, int nj, int C, int F, int H, int W, int row_limit, int blend_extent,
                                     int t_limit, int t_blend_extent, void* out, void* stream_) {
  if (!tile_ptrs || !th || !tw || !tlen || !tf0 || !out) return YB_ERR_ARG;
  if (nt <= 0 || ni <= 0 || nj <= 0 || C <= 0 || F <= 0 || H <= 0 || W <= 0) return YB_ERR_ARG;
  if ((ni > 1 || nj > 1) && (row_limit <= 0 || blend_extent <= 0)) return YB_ERR_ARG;
  if (nt > 1 && (t_limit <= 0 || t_blend_extent <= 0)) return YB_ERR_ARG;
  TileAsm a;
  a.ptr = reinterpret_cast<const float* const*>(tile_ptrs);
  a.th = th; a.tw = tw; a.tlen = tlen; a.tf0 = tf0;
  a.nt = nt; a.ni = ni; a.nj = nj; a.C = C; a.F = F; a.H = H; a.W = W;
  a.rl = (ni > 1 || nj > 1) ? row_limit : 0;
  a.E = blend_extent;
  a.tl = t_limit;
  a.Et = t_blend_extent;
  vae_assemble_tiles_kernel<<<grid_for(static_cast<long long>(C) * F * H * W), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      a, static_cast<float*>(out));
  return check_launch("vae_assemble_tiles");
}

extern "C" int yb_vae_rms_act(const void* x, long long ldx, void* out, const void* gamma, int T, int Hs, int Ws, int C,
                              int Cp, int up, int silu, void* stream_) {
  if (!x || !out || T <= 0 || Hs <= 0 || Ws <= 0 || C <= 0) return YB_ERR_ARG;
  if (C % 8 != 0 || Cp % 8 != 0 || Cp < C || (up != 1 && up != 2)) return YB_ERR_SHAPE;
  if ((ldx % 8) || (reinterpret_cast<uintptr_t>(x) & 0xF) || (reinterpret_cast<uintptr_t>(out) & 0xF)) return YB_ERR_ALIGNMENT;
  if (C > 1024) return YB_ERR_SHAPE;
  if (gamma && (reinterpret_cast<uintptr_t>(gamma) & 0xF)) return YB_ERR_ALIGNMENT;
  const long long nvox = static_cast<long long>(T) * Hs * up * Ws * up;
  if (nvox > 0x7fffffffLL - (1LL << 24)) return YB_ERR_SHAPE;                      // 32-bit voxel indices in the kernel
  const int nch = C <= 256 ? 1 : (C <= 512 ? 2 : 4);
  const int g = nch > 1 ? 32 : (Cp <= 64 ? 8 : (Cp <= 128 ? 16 : 32));         // lanes per voxel
  const int per_block = 8 * (4 / nch) * (32 / g);
  long long blocks = (nvox + per_block - 1) / per_block;
  if (blocks > static_cast<long long>(sm_count()) * 32) blocks = static_cast<long long>(sm_count()) * 32;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
#define YB_RMS_LAUNCH(NCH, G)                                                                                        \
  rms_act_kernel<NCH, G><<<static_cast<int>(blocks), 256, 0, st>>>(static_cast<const __nv_bfloat16*>(x), ldx,         \
                                                                  static_cast<__nv_bfloat16*>(out),                    \
                                                                  static_cast<const float*>(gamma), T, Hs, Ws, C, Cp, up, silu)
  if (nch == 4) YB_RMS_LAUNCH(4, 32);
  else if (nch == 2) YB_RMS_LAUNCH(2, 32);
  else if (g == 32) YB_RMS_LAUNCH(1, 32);
  else if (g == 16) YB_RMS_LAUNCH(1, 16);
  else YB_RMS_LAUNCH(1, 8);
#undef YB_RMS_LAUNCH
  return check_launch("vae_rms_act");
}

extern "C" int yb_vae_rms_act_fp8(const void* x, long long ldx, void* out, void* out_scale, const void* gamma, int T, int Hs, int Ws,
                                  int C, int Cp, int up, int silu, void* stream_) {
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

static int dupup_launch(void* main_, const void* x, int Ts, int Hs, int Ws, int in_c, int out_c, int ft, int fs, bool first,
                        void* stream_) {
  if (!main_ || !x || Ts <= 0 || Hs <= 0 || Ws <= 0 || in_c <= 0 || out_c <= 0 || ft < 1 || fs < 1) return YB_ERR_ARG;
  if ((out_c * ft * fs * fs) % in_c != 0 || out_c % 8 != 0) return YB_ERR_SHAPE;
  if (reinterpret_cast<uintptr_t>(main_) & 0xF) return YB_ERR_ALIGNMENT;
  const int drop = first ? ft - 1 : 0;
  if (static_cast<long long>(ft * Ts - drop) * Hs * fs * Ws * fs > 0x7fffffffLL) return YB_ERR_SHAPE;
  const long long total = static_cast<long long>(ft * Ts - drop) * Hs * fs * Ws * fs * (out_c / 8);
  dupup_add_kernel<<<grid_for(total), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<__nv_bfloat16*>(main_), static_cast<const __nv_bfloat16*>(x), Ts, Hs, Ws, in_c, out_c, ft, fs, drop);
  return check_launch("vae_dupup_add");
}

extern "C" int yb_vae_dupup_add(void* main_, const void* x, int Ts, int Hs, int Ws, int in_c, int out_c, int ft, int fs,
                                void* stream_) {
  return dupup_launch(main_, x, Ts, Hs, Ws, in_c, out_c, ft, fs, true, stream_);
}

extern "C" int yb_vae_dupup_add_cont(void* main_, const void* x, int Ts, int Hs, int Ws, int in_c, int out_c, int ft, int fs,
                                     void* stream_) {
  return dupup_launch(main_, x, Ts, Hs, Ws, in_c, out_c, ft, fs, false, stream_);
}

extern "C" int yb_vae_avgdown_add(void* main_, const void* x, int T, int H, int W, int in_c, int out_c, int ft, int fs,
                                  void* stream_) {
  if (!main_ || !x || T <= 0 || H <= 0 || W <= 0 || in_c <= 0 || out_c <= 0 || ft < 1 || fs < 1) return YB_ERR_ARG;
  if ((in_c * ft * fs * fs) % out_c != 0 || out_c % 8 != 0 || H % fs != 0 || W % fs != 0) return YB_ERR_SHAPE;
  if (reinterpret_cast<uintptr_t>(main_) & 0xF) return YB_ERR_ALIGNMENT;
  const long long To = (T + (ft - T % ft) % ft) / ft;
  if (To * (H / fs) * (W / fs) > 0x7fffffffLL) return YB_ERR_SHAPE;
  const long long total = To * (H / fs) * (W / fs) * (out_c / 8);
  avgdown_add_kernel<<<grid_for(total), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<__nv_bfloat16*>(main_), static_cast<const __nv_bfloat16*>(x), T, H, W, in_c, out_c, ft, fs);
  return check_launch("vae_avgdown_add");
}

extern "C" int yb_vae_patchify2_bf16_win(const void* video, long long plane, void* out, long long ldo, int T, int H, int W,
                                         void* stream_) {
  if (!video || !out || T <= 0 || H <= 0 || W <= 0 || ldo < 12) return YB_ERR_ARG;
  if ((H % 2) || (W % 2)) return YB_ERR_SHAPE;
  if (plane < static_cast<long long>(T) * H * W) return YB_ERR_ARG;
  if ((reinterpret_cast<uintptr_t>(video) & 0x7) || (plane % 2)) return YB_ERR_ALIGNMENT;
  patchify2_bf16_kernel<<<grid_for(static_cast<long long>(T) * (H / 2) * (W / 2)), 256, 0,
                          reinterpret_cast<cudaStream_t>(stream_)>>>(static_cast<const float*>(video),
                                                                     static_cast<__nv_bfloat16*>(out), ldo, T, H, W, plane);
  return check_launch("vae_patchify2_bf16");
}

extern "C" int yb_vae_patchify2_bf16(const void* video, void* out, long long ldo, int T, int H, int W, void* stream_) {
  return yb_vae_patchify2_bf16_win(video, static_cast<long long>(T) * H * W, out, ldo, T, H, W, stream_);
}

extern "C" int yb_vae_unpatchify2_clamp_win(const void* y, long long ldy, void* out, long long plane, int T, int H, int W,
                                            void* stream_) {
  if (!y || !out || T <= 0 || H <= 0 || W <= 0 || ldy < 12 || plane < 4LL * T * H * W) return YB_ERR_ARG;
  unpatchify2_clamp_kernel<<<grid_for(12LL * T * H * W), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(y), ldy, static_cast<float*>(out), T, H, W, plane);
  return check_launch("vae_unpatchify2_clamp");
}

extern "C" int yb_vae_unpatchify2_clamp(const void* y, long long ldy, void* out, int T, int H, int W, void* stream_) {
  return yb_vae_unpatchify2_clamp_win(y, ldy, out, 4LL * T * H * W, T, H, W, stream_);
}

extern "C" int yb_nhwc_to_nchw_f32_clamp_win(const void* x, long long ldx, void* out, long long plane, long long N, int Cn,
                                             float lo, float hi, void* stream_) {
  if (!x || !out || N <= 0 || Cn <= 0 || ldx < Cn || plane < N || !(lo <= hi)) return YB_ERR_ARG;
  nhwc_to_nchw_kernel<<<grid_for(N * Cn), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(x), ldx, static_cast<float*>(out), N, Cn, lo, hi, plane);
  return check_launch("nhwc_to_nchw_clamp");
}

extern "C" int yb_vae_frame_match(const void* kept, int t_kept, const void* x, int t, int C, long long frame_elems,
                                  int elem_bytes, int* result, void* stream_) {
  if (!x || !result || t <= 0 || t_kept < 0 || C <= 0 || frame_elems <= 0 || (t_kept > 0 && !kept)) return YB_ERR_ARG;
  if (elem_bytes != 1 && elem_bytes != 2 && elem_bytes != 4 && elem_bytes != 8) return YB_ERR_ARG;
  if (reinterpret_cast<uintptr_t>(result) & 0x3) return YB_ERR_ALIGNMENT;
  const long long frame_bytes = frame_elems * elem_bytes;
  const uintptr_t addr = reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(t_kept > 0 ? kept : x) |
                         static_cast<uintptr_t>(frame_bytes);
  const int vec = (addr & 0xF) == 0 ? 16 : (addr & 0x7) == 0 ? 8 : (addr & 0x3) == 0 ? 4 : (addr & 0x1) == 0 ? 2 : 1;
  const long long rows = static_cast<long long>(C) * t, nvec = frame_bytes / vec;
  const long long items = rows * ((nvec + FM_VEC_PER_THREAD * 256 - 1) / (FM_VEC_PER_THREAD * 256));
  const long long cap = static_cast<long long>(sm_count()) * 8;
  const int grid = static_cast<int>(items < cap ? items : cap);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  frame_match_init_kernel<<<1, 1, 0, st>>>(result, t_kept < t ? t_kept : t);
#define YB_FM_LAUNCH(V)                                                                                                  \
  frame_match_kernel<V><<<grid, 256, 0, st>>>(static_cast<const V*>(kept), t_kept, static_cast<const V*>(x), t, rows, nvec, \
                                              result)
  if (vec == 16) YB_FM_LAUNCH(uint4);
  else if (vec == 8) YB_FM_LAUNCH(unsigned long long);
  else if (vec == 4) YB_FM_LAUNCH(unsigned int);
  else if (vec == 2) YB_FM_LAUNCH(unsigned short);
  else YB_FM_LAUNCH(unsigned char);
#undef YB_FM_LAUNCH
  return check_launch("vae_frame_match");
}

// ---------------------------------------------------------------------------------------------------------
// Row-band forms (include/yume_b200_vae_rows.h)
// ---------------------------------------------------------------------------------------------------------
extern "C" int yb_vae_rms_act_rows(const void* x, long long ldx, void* out, void* send, const void* gamma, int T, int Hs, int Ws,
                                   int C, int Cp, int up, int silu, void* stream_) {
  if (!x || !out || T <= 0 || Hs <= 0 || Ws <= 0 || C <= 0) return YB_ERR_ARG;
  if (C % 8 != 0 || Cp % 8 != 0 || Cp < C || (up != 1 && up != 2)) return YB_ERR_SHAPE;
  if ((ldx % 8) || (reinterpret_cast<uintptr_t>(x) & 0xF) || (reinterpret_cast<uintptr_t>(out) & 0xF) ||
      (reinterpret_cast<uintptr_t>(send) & 0xF))
    return YB_ERR_ALIGNMENT;
  if (C > 1024) return YB_ERR_SHAPE;
  if (gamma && (reinterpret_cast<uintptr_t>(gamma) & 0xF)) return YB_ERR_ALIGNMENT;
  const long long nvox = static_cast<long long>(T) * (Hs * up + 2) * Ws * up;   // the buffer's voxels: 32-bit indices
  if (nvox > 0x7fffffffLL - (1LL << 24)) return YB_ERR_SHAPE;
  // the (NCH, G) instance and grid of yb_vae_rms_act for the same arguments
  const int nch = C <= 256 ? 1 : (C <= 512 ? 2 : 4);
  const int g = nch > 1 ? 32 : (Cp <= 64 ? 8 : (Cp <= 128 ? 16 : 32));
  const int per_block = 8 * (4 / nch) * (32 / g);
  long long blocks = (static_cast<long long>(T) * Hs * up * Ws * up + per_block - 1) / per_block;
  if (blocks > static_cast<long long>(sm_count()) * 32) blocks = static_cast<long long>(sm_count()) * 32;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
#define YB_RMS_ROWS_LAUNCH(NCH, G)                                                                                         \
  rms_act_kernel<NCH, G, true><<<static_cast<int>(blocks), 256, 0, st>>>(                                                  \
      static_cast<const __nv_bfloat16*>(x), ldx, static_cast<__nv_bfloat16*>(out), static_cast<const float*>(gamma), T, Hs, \
      Ws, C, Cp, up, silu, static_cast<__nv_bfloat16*>(send))
  if (nch == 4) YB_RMS_ROWS_LAUNCH(4, 32);
  else if (nch == 2) YB_RMS_ROWS_LAUNCH(2, 32);
  else if (g == 32) YB_RMS_ROWS_LAUNCH(1, 32);
  else if (g == 16) YB_RMS_ROWS_LAUNCH(1, 16);
  else YB_RMS_ROWS_LAUNCH(1, 8);
#undef YB_RMS_ROWS_LAUNCH
  return check_launch("vae_rms_act_rows");
}

static int rows_glue_check(const void* a, const void* b, const void* c, int T, int Hs, long long row_bytes) {
  if (T <= 0 || Hs <= 0 || row_bytes <= 0) return YB_ERR_ARG;
  if ((row_bytes % 16) || (reinterpret_cast<uintptr_t>(a) & 0xF) || (reinterpret_cast<uintptr_t>(b) & 0xF) ||
      (reinterpret_cast<uintptr_t>(c) & 0xF))
    return YB_ERR_ALIGNMENT;
  return YB_OK;
}

extern "C" int yb_vae_rows_pack(const void* buf, void* send, int T, int Hs, long long row_bytes, void* stream_) {
  if (!buf || !send) return YB_ERR_ARG;
  if (int rc = rows_glue_check(buf, send, nullptr, T, Hs, row_bytes)) return rc;
  rows_pack_kernel<<<grid_for(2LL * T * (row_bytes / 16)), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const uint4*>(buf), static_cast<uint4*>(send), T, Hs, row_bytes / 16);
  return check_launch("vae_rows_pack");
}

extern "C" int yb_vae_rows_unpack(const void* recv_top, const void* recv_bot, void* buf, int T, int Hs, long long row_bytes,
                                  void* stream_) {
  if (!buf) return YB_ERR_ARG;
  if (int rc = rows_glue_check(recv_top, recv_bot, buf, T, Hs, row_bytes)) return rc;
  rows_unpack_kernel<<<grid_for(2LL * T * (row_bytes / 16)), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const uint4*>(recv_top), static_cast<const uint4*>(recv_bot), static_cast<uint4*>(buf), T, Hs, row_bytes / 16);
  return check_launch("vae_rows_unpack");
}

extern "C" int yb_vae_unpatchify2_clamp_rows(const void* y, long long ldy, void* out, long long plane, long long frame, int T,
                                             int Hs, int W, void* stream_) {
  if (!y || !out || T <= 0 || Hs <= 0 || W <= 0 || ldy < 12 || frame < 4LL * Hs * W || plane < frame * T) return YB_ERR_ARG;
  unpatchify2_clamp_rows_kernel<<<grid_for(12LL * T * Hs * W), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(y), ldy, static_cast<float*>(out), T, Hs, W, plane, frame);
  return check_launch("vae_unpatchify2_clamp_rows");
}

extern "C" int yb_nhwc_to_nchw_f32_clamp_rows(const void* x, long long ldx, void* out, long long plane, long long frame, int T,
                                              int Hs, int W, int Cn, float lo, float hi, void* stream_) {
  if (!x || !out || T <= 0 || Hs <= 0 || W <= 0 || Cn <= 0 || ldx < Cn || frame < static_cast<long long>(Hs) * W ||
      plane < frame * T || !(lo <= hi))
    return YB_ERR_ARG;
  nhwc_to_nchw_rows_kernel<<<grid_for(static_cast<long long>(T) * Hs * W * Cn), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      static_cast<const float*>(x), ldx, static_cast<float*>(out), T, Hs, W, Cn, lo, hi, plane, frame);
  return check_launch("nhwc_to_nchw_clamp_rows");
}

// ---------------------------------------------------------------------------------------------------------
// Band readers of the row-parallel encode (include/yume_b200_vae_rows_enc.h)
// ---------------------------------------------------------------------------------------------------------
static int rows_reader_check(const void* src, long long plane, const void* out, int ldo, int T, int H, int W, int rows, int r0,
                             int hs) {
  if (!src || !out || T <= 0 || H <= 0 || W <= 0 || hs <= 0 || r0 < 0 || r0 + hs > rows) return YB_ERR_ARG;
  if (plane < static_cast<long long>(T) * H * W) return YB_ERR_ARG;
  if ((ldo % 8) || (reinterpret_cast<uintptr_t>(out) & 0xF)) return YB_ERR_ALIGNMENT;
  return YB_OK;
}

extern "C" int yb_vae_patchify2_bf16_rows(const void* video, long long plane, void* out, int ldo, int T, int H, int W, int r0,
                                          int hs, void* stream_) {
  if (H <= 0 || W <= 0 || ldo < 12) return YB_ERR_ARG;
  if ((H % 2) || (W % 2)) return YB_ERR_SHAPE;
  if (int rc = rows_reader_check(video, plane, out, ldo, T, H, W, H / 2, r0, hs)) return rc;
  if ((reinterpret_cast<uintptr_t>(video) & 0x7) || (plane % 2)) return YB_ERR_ALIGNMENT;
  patchify2_bf16_rows_kernel<<<grid_for(static_cast<long long>(T) * (hs + 2) * (W / 2)), 256, 0,
                               reinterpret_cast<cudaStream_t>(stream_)>>>(static_cast<const float*>(video),
                                                                          static_cast<__nv_bfloat16*>(out), ldo, T, H, W, plane,
                                                                          r0, hs);
  return check_launch("vae_patchify2_bf16_rows");
}

extern "C" int yb_nchw_to_nhwc_bf16_rows(const void* x, long long plane, void* out, int ldo, int T, int H, int W, int Cn, int r0,
                                         int hs, void* stream_) {
  if (Cn <= 0 || ldo < Cn) return YB_ERR_ARG;
  if (int rc = rows_reader_check(x, plane, out, ldo, T, H, W, H, r0, hs)) return rc;
  nchw_to_nhwc_rows_kernel<<<grid_for(static_cast<long long>(T) * (hs + 2) * W * ldo), 256, 0,
                             reinterpret_cast<cudaStream_t>(stream_)>>>(static_cast<const float*>(x),
                                                                        static_cast<__nv_bfloat16*>(out), ldo, T, H, W, Cn, plane,
                                                                        r0, hs);
  return check_launch("nchw_to_nhwc_bf16_rows");
}
