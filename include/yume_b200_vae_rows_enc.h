/* yume_b200_vae_rows_enc.h — C ABI of the row-band forms of the Wan VAE ENCODE kernels in libyume_b200.so (conventions as
 * include/yume_b200.h: device pointers, `stream` a cudaStream_t as void*, no allocation, no synchronisation, capture-safe
 * launches, 0 or a negative YB_ERR_* code).
 *
 * Row-parallel encode (WanVaeEncoder.enable_row_parallel): P ranks split the LATENT's H rows into bands, rank r owning rows
 * [floor(rH/P), floor((r+1)H/P)) and, at every level above the latent, those rows times the level's scale. Every stride-2 level
 * halves a band exactly, so a band is a whole set of rows at every level. The unit-stride convs (kh = 3) read band buffers
 * [t_hist + T, Hs + 2, W, Cp] through yb_conv3d_rows (include/yume_b200_vae_rows.h); the forms here are the rest:
 *   - the video readers, which write a band buffer's rows AND both halo rows straight from the whole video that every rank holds
 *     (no exchange), zeros beyond the image's top and bottom edge;
 *   - the strided Resample conv (ZeroPad2d((0,1,0,1)) + Conv2d 3x3 stride 2), whose output rows [a, b) read input rows 2a .. 2b:
 *     only the row BELOW the band, the first row of the band below, or zeros on the last band (the reference's pad row).
 *
 * Bit identity: the readers convert each element exactly as their _win twins; the strided conv never fuses the kw taps and sums
 * every output voxel's products in the same (tap, channel block) order as the full-height yb_conv3d_causal(stride_hw = 2). A
 * row-parallel encode is therefore equal bit for bit to the one-GPU encode.
 */
#ifndef YUME_B200_VAE_ROWS_ENC_H_
#define YUME_B200_VAE_ROWS_ENC_H_

#include "yume_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Strided row-halo conv: the Resample downsample2d of a band. `xpad` is a band buffer [T, H + 2, W, Cp] with H the band's INPUT
 * rows: rows 1 .. H the band, row H + 1 the first row of the band below (zeros on the last band), row 0 not read. Output rows
 * (t * H/2 + h) * W/2 + w, h < H/2, as the full-height yb_conv3d_causal(stride_hw = 2) writes them for its rows. W keeps the
 * out-of-bounds zero fill (the right pad column). Taps (1,3,3), stride_hw = 2, stride_t = 1, no history; H even and
 * oob_zero_pad == 1, else YB_ERR_ARG. Other constraints: those of yb_conv3d_causal. */
int yb_conv3d_rows_down(const yb_conv3d_args* args, void* stream);

/* Band readers of the encoder's input. The source is a frame window of the whole video: channel 0, the window's frame 0, row 0;
 * channel planes `plane` elements apart, frames H * W apart (H x W the whole video's frame). They write the T frames of a band
 * buffer out [T, hs + 2, Wo, ldo] (bf16, contiguous): buffer row j is image row r0 - 1 + j of the reader's output level, all
 * zero when that row lies outside the image; columns beyond the data channels are zero.
 *   yb_vae_patchify2_bf16_rows: video f32 [3, T, H, W] -> the patchified rows (12 channels, Wo = W / 2, rows of H / 2), element
 *                               for element yb_vae_patchify2_bf16_win; ldo >= 12
 *   yb_nchw_to_nhwc_bf16_rows:  x f32 [Cn, T, H, W] -> channels-last rows (Wo = W, rows of H), element for element
 *                               yb_nchw_to_nhwc_bf16_win; ldo >= Cn
 * Constraints: 0 <= r0, hs >= 1, r0 + hs <= the level's rows, plane >= T * H * W, ldo % 8 == 0 and out 16-byte aligned
 * (YB_ERR_ALIGNMENT); patchify: H, W even (YB_ERR_SHAPE), video 8-byte aligned. */
int yb_vae_patchify2_bf16_rows(const void* video, long long plane, void* out, int ldo, int T, int H, int W, int r0, int hs,
                               void* stream);
int yb_nchw_to_nhwc_bf16_rows(const void* x, long long plane, void* out, int ldo, int T, int H, int W, int Cn, int r0, int hs,
                              void* stream);

#ifdef __cplusplus
}
#endif
#endif /* YUME_B200_VAE_ROWS_ENC_H_ */
