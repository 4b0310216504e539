/* yume_b200_clip.h — C ABI of the CLIP vision-encoder input kernel in libyume_b200.so (conventions as include/yume_b200.h:
 * device pointers, `stream` a cudaStream_t as void*, no allocation, no synchronisation, 0 or a negative YB_ERR_* code).
 *
 * The encoder's transformer runs on the entry points of include/yume_b200.h (yb_ln_modulate, yb_gemm_bf16, yb_attention,
 * yb_patchify); this header adds the one step they do not cover.
 */
#ifndef YUME_B200_CLIP_H_
#define YUME_B200_CLIP_H_

#include "yume_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------------
 * Bicubic resize + CLIP Normalize: the preprocessing of CLIPModel.visual (wan/modules/clip.py:529-537),
 *   F.interpolate(u, size=(S, S), mode='bicubic', align_corners=False)   (no antialias, fp32)
 *   .mul_(0.5).add_(0.5)                                                 ([-1, 1] -> [0, 1])
 *   T.Normalize(mean, std)                                               (sub_(mean).div_(std) per channel)
 *   x     f32 [C, H, W], element strides sc, sh, sw (any layout: the [3, 1, H, W] image is read in place)
 *   out   f32 [C, S, S] contiguous
 *   mean, std  f32 [C] device arrays
 * Arithmetic of PyTorch's CUDA upsample_bicubic2d: scale = (float)H / S (and W / S); source coordinate
 * fmaf(scale, dst + 0.5f, -0.5f), not clamped; Keys coefficients with A = -0.75 from t = src - floorf(src); the four taps of
 * each axis clamped to the border; the four rows are interpolated along x, then the four results along y. H == S and W == S
 * copies. Then v * 0.5f + 0.5f, - mean[c], / std[c], each rounded separately (IEEE division).
 * Constraints: C, H, W, S > 0.
 * ------------------------------------------------------------------------------------------- */
int yb_resize_bicubic_normalize(const void* x, long long sc, long long sh, long long sw, int C, int H, int W, void* out,
                                int S, const void* mean, const void* std, void* stream);

#ifdef __cplusplus
}
#endif

#endif  // YUME_B200_CLIP_H_
