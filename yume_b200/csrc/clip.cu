// clip.cu — the input step of the CLIP ViT-H/14 image encoder (wan/modules/clip.py:527-542): bicubic resize to the model's
// image size and the CLIP Normalize, in one pass. The transformer itself runs on the GEMM / LayerNorm / attention kernels.
#include <cuda_runtime.h>

#include "../../include/yume_b200_clip.h"
#include "yb_host.h"

namespace {

// Keys cubic convolution with A = -0.75, written as PyTorch's ATen/native/cuda/UpSample.cuh writes it so that nvcc evaluates
// (and contracts) it the same way: |x| <= 1 and 1 < |x| < 2.
__device__ __forceinline__ float cubic_convolution1(float x, float A) { return ((A + 2) * x - (A + 3)) * x * x + 1; }
__device__ __forceinline__ float cubic_convolution2(float x, float A) { return ((A * x - 5 * A) * x + 8 * A) * x - 4 * A; }

__device__ __forceinline__ float cubic_interp1d(float x0, float x1, float x2, float x3, float t) {
  const float A = -0.75f;
  const float c0 = cubic_convolution2(t + 1.0f, A);
  const float c1 = cubic_convolution1(t, A);
  const float x2t = 1.0f - t;
  const float c2 = cubic_convolution1(x2t, A);
  const float c3 = cubic_convolution2(x2t + 1.0f, A);
  return x0 * c0 + x1 * c1 + x2 * c2 + x3 * c3;
}

// one thread per output pixel, all C channels (the coordinate math is shared)
__global__ void resize_bicubic_normalize_kernel(const float* __restrict__ x, long long sc, long long sh, long long sw, int C,
                                                int H, int W, float* __restrict__ out, int S, float scale_h, float scale_w,
                                                const float* __restrict__ mean, const float* __restrict__ std) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= S * S) return;
  const int ox = idx % S, oy = idx / S;
  const bool copy = (H == S && W == S);
  // source coordinates: scale * (dst + 0.5) - 0.5, one rounding (the FMA nvcc forms from PyTorch's expression), not clamped
  const float real_x = __fmaf_rn(scale_w, static_cast<float>(ox) + 0.5f, -0.5f);
  const float real_y = __fmaf_rn(scale_h, static_cast<float>(oy) + 0.5f, -0.5f);
  const int in_x = static_cast<int>(floorf(real_x)), in_y = static_cast<int>(floorf(real_y));
  const float t_x = real_x - static_cast<float>(in_x), t_y = real_y - static_cast<float>(in_y);
  int xs[4], ys[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {                    // taps clamped to the border
    xs[k] = max(min(in_x - 1 + k, W - 1), 0);
    ys[k] = max(min(in_y - 1 + k, H - 1), 0);
  }
  for (int c = 0; c < C; ++c) {
    const float* xc = x + c * sc;
    float v;
    if (copy) {
      v = xc[oy * sh + ox * sw];
    } else {
      float r[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float* row = xc + ys[k] * sh;
        r[k] = cubic_interp1d(row[xs[0] * sw], row[xs[1] * sw], row[xs[2] * sw], row[xs[3] * sw], t_x);
      }
      v = cubic_interp1d(r[0], r[1], r[2], r[3], t_y);
    }
    v = __fadd_rn(__fmul_rn(v, 0.5f), 0.5f);     // mul_(0.5).add_(0.5)
    v = __fdiv_rn(__fsub_rn(v, mean[c]), std[c]);  // Normalize: sub_(mean).div_(std)
    out[(static_cast<long long>(c) * S + oy) * S + ox] = v;
  }
}

}  // namespace

extern "C" int yb_resize_bicubic_normalize(const void* x, long long sc, long long sh, long long sw, int C, int H, int W,
                                           void* out, int S, const void* mean, const void* std, void* stream) {
  if (!x || !out || !mean || !std || C <= 0 || H <= 0 || W <= 0 || S <= 0) return YB_ERR_ARG;
  // area_pixel_compute_scale (align_corners = false, no scale_factor): input_size / output_size in float
  const float scale_h = static_cast<float>(H) / static_cast<float>(S);
  const float scale_w = static_cast<float>(W) / static_cast<float>(S);
  const int threads = 256;
  const int blocks = (S * S + threads - 1) / threads;
  resize_bicubic_normalize_kernel<<<blocks, threads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      static_cast<const float*>(x), sc, sh, sw, C, H, W, static_cast<float*>(out), S, scale_h, scale_w,
      static_cast<const float*>(mean), static_cast<const float*>(std));
  return yb::check_launch("resize_bicubic_normalize");
}
