/* yume_b200_stream.h — C ABI of the chunk-streaming forms of the Wan VAE kernels in libyume_b200.so (conventions as
 * include/yume_b200.h: device pointers, `stream` a cudaStream_t as void*, no allocation, no synchronisation, capture-safe
 * launches, 0 or a negative YB_ERR_* code).
 *
 * The reference decodes one latent frame per Decoder3d call and hands every CausalConv3d the last CACHE_T = 2 frames of its
 * input from the previous call (wan/modules/vae.py:14, 544-568; wan23/modules/vae2_2.py:831-860), so its memory does not grow
 * with the video. The decoders here split the latent into chunks of any length and carry the same state between chunks; these
 * entry points are the forms a chunk after the first needs. The encoders stream the same way: the reference encodes frame 0,
 * then 4 frames per Encoder3d call (wan/modules/vae.py:515-542; vae2_2.py:796-829); here the first chunk holds 1 + 4a frames and
 * every later chunk 4b. A whole sequence in one chunk uses only include/yume_b200.h.
 */
#ifndef YUME_B200_STREAM_H_
#define YUME_B200_STREAM_H_

#include "yume_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* History form of yb_conv3d_causal (needs oob_zero_pad = 1). `xpad` is [t_hist + T, H, W, Cp]: its first t_hist frames are the
 * carried input frames of the previous chunk and take the place of the causal zero padding in time; H and W keep the
 * out-of-bounds zero fill. T is the number of NEW frames.
 *   unit stride:  t_hist = kt - 1; output frame t (of T) reads buffer frames t .. t + kt - 1
 *   stride_t = 2: t_hist = 1 (the frame the encoder's time_conv carries, vae2_2.py:158-170); To = (t_hist + T - kt) / 2 + 1
 * Every other field means what it means for yb_conv3d_causal and takes the same tile plan for the same output extents, so
 * each output voxel sums the same products in the same order as the one-pass launch over the whole sequence. */
int yb_conv3d_causal_hist(const yb_conv3d_args* args, int t_hist, void* stream);

/* yb_vae_dupup_add for a chunk after the first: no duplicated frame is dropped (DupUp3D's `first_chunk`, vae2_2.py:376-418,
 * 495-503). main bf16 [ft*Ts, Hs*fs, Ws*fs, out_c], x bf16 [Ts, Hs, Ws, in_c], both dense. */
int yb_vae_dupup_add_cont(void* main_, const void* x, int Ts, int Hs, int Ws, int in_c, int out_c, int ft, int fs, void* stream);

/* Window forms of the two decoder tails: the chunk's T frames are written into a frame window of the whole video. `out` points
 * at frame 0 of the window in channel 0; channel planes are `plane` elements apart (the whole video's frames x rows x columns).
 *   yb_vae_unpatchify2_clamp_win: as yb_vae_unpatchify2_clamp; plane >= 4*T*H*W
 *   yb_nhwc_to_nchw_f32_clamp_win: as yb_nhwc_to_nchw_f32_clamp; plane >= N */
int yb_vae_unpatchify2_clamp_win(const void* y, long long ldy, void* out, long long plane, int T, int H, int W, void* stream);
int yb_nhwc_to_nchw_f32_clamp_win(const void* x, long long ldx, void* out, long long plane, long long N, int Cn, float lo,
                                  float hi, void* stream);
/* (The encoders write their mu chunk with yb_nhwc_to_nchw_f32_clamp_win and lo = -inf, hi = +inf: no clamp, the arithmetic of
 * yb_nhwc_to_nchw_f32.) */

/* Window forms of the two encoder inputs: the chunk's T frames are read from a frame window of the whole video. `video` / `x`
 * points at frame 0 of the window in channel 0; channel planes are `plane` elements apart.
 *   yb_vae_patchify2_bf16_win: as yb_vae_patchify2_bf16; plane >= T*H*W, even
 *   yb_nchw_to_nhwc_bf16_win: as yb_nchw_to_nhwc_bf16 (x [Cn, N] with N = T*H*W new voxels); plane >= N */
int yb_vae_patchify2_bf16_win(const void* video, long long plane, void* out, long long ldo, int T, int H, int W, void* stream);
int yb_nchw_to_nhwc_bf16_win(const void* x, long long plane, void* out, long long N, int Cn, int ldo, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* YUME_B200_STREAM_H_ */
