/* yume_b200_vae_rows.h — C ABI of the row-band forms of the Wan VAE decode kernels in libyume_b200.so (conventions as
 * include/yume_b200.h: device pointers, `stream` a cudaStream_t as void*, no allocation, no synchronisation, capture-safe
 * launches, 0 or a negative YB_ERR_* code).
 *
 * Row-parallel decode (WanVaeDecoder.enable_row_parallel): P ranks split the latent's H rows into bands, rank r owning rows
 * [floor(rH/P), floor((r+1)H/P)). Every 2x upsample doubles a band, so a band is a whole set of rows at every level. Everything
 * in the decoder is per voxel or per row except
 *   - the spatial convs, all with kh = 3: a rank needs one row of each neighbour's band (a "halo" row) on each side;
 *   - the per-frame mid attention, which runs on the gathered full frames (see DESIGN.md §6).
 * A conv input of a band is a BAND BUFFER [t_hist + T, Hs + 2, W, Cp]: rows 1 .. Hs are the rank's own rows, row 0 is the last
 * row of the band above and row Hs + 1 the first row of the band below, or zeros at the image's top and bottom edge (the conv's
 * zero padding in H). The forms here write, exchange and read those buffers; the send / receive buffers of the exchange are
 * [2, T, W, Cp]: [0] the top row, [1] the bottom row of the T frames.
 *
 * Bit identity: the row-halo conv takes the tile plan yb_conv3d_plan gives for its own output extents; told whether the
 * full-height launch fuses the kw taps, it sums, for every output voxel, the same products in the same (tap, channel block) order
 * as that launch. The other forms move or compute each element exactly as their full-height twins. A row-parallel decode is
 * therefore equal bit for bit to the one-GPU decode.
 */
#ifndef YUME_B200_VAE_ROWS_H_
#define YUME_B200_VAE_ROWS_H_

#include "yume_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Row-halo form of yb_conv3d_causal / yb_conv3d_causal_hist (oob_zero_pad = 1, kh = 3, unit stride). `xpad` is the band buffer
 * [t_hist + T, H + 2, W, Cp] with H the band's row count (the OUTPUT rows): output row h reads buffer rows h .. h + 2, with no
 * zero fill in H. W keeps the out-of-bounds zero fill; time keeps the causal zero fill (t_hist = 0) or the t_hist = kt - 1
 * carried frames in front. Covers taps (3,3,3) and (1,3,3) and the BF16, F32 and RES_BF16 epilogues. Output rows
 * (t * H + h) * W + w, as the full-height launch writes them for its rows. The kw-fused and the unfused sum (yb_conv3d_args.fuse_w)
 * may round differently: for the full-height launch's bits pass fuse_w = 2 when yb_conv3d_plan reports that launch fused, else 1.
 * Constraints: those of yb_conv3d_causal_hist; kh == 3, stride 1 and oob_zero_pad == 1 (YB_ERR_ARG). */
int yb_conv3d_rows(const yb_conv3d_args* args, int t_hist, void* stream);

/* Band form of yb_vae_rms_act: x bf16 [T * Hs * Ws, C] (row stride ldx) -> rows 1 .. Hs * up of out, a band buffer
 * [T, Hs * up + 2, Ws * up, Cp] (the T new frames; rows 0 and Hs * up + 1 are not written). up = 2 is the nearest-exact 2x
 * upsample. send (may be NULL): [2, T, Ws * up, Cp], receives the first and the last written row of every frame, the values
 * written into out (the rows the neighbours need). Constraints: those of yb_vae_rms_act; send 16-byte aligned. */
int yb_vae_rms_act_rows(const void* x, long long ldx, void* out, void* send, const void* gamma, int T, int Hs, int Ws, int C,
                        int Cp, int up, int silu, void* stream);

/* Halo exchange glue on T band-buffer frames [T, Hs + 2, row_bytes] (buf: the first of the T frames):
 *   yb_vae_rows_pack:   send [2, T, row_bytes] = rows 1 and Hs of every frame (for a buffer not written by yb_vae_rms_act_rows)
 *   yb_vae_rows_unpack: row 0 = recv_top[t], row Hs + 1 = recv_bot[t]; a NULL source writes zeros (the image's edge)
 * row_bytes % 16 == 0 and every pointer 16-byte aligned (YB_ERR_ALIGNMENT). */
int yb_vae_rows_pack(const void* buf, void* send, int T, int Hs, long long row_bytes, void* stream);
int yb_vae_rows_unpack(const void* recv_top, const void* recv_bot, void* buf, int T, int Hs, long long row_bytes, void* stream);

/* Row-band forms of the two decoder tails: the chunk's T frames x Hs band rows are written at a row of a frame window of the whole
 * video. `out` points at channel 0, the window's frame 0, the band's first output row; channel planes are `plane` and frames
 * `frame` elements apart (the whole video's frames x rows x columns, and rows x columns).
 *   yb_vae_unpatchify2_clamp_rows: y f32 [T * Hs * W, ldy] -> 3 channels x T frames x 2Hs rows x 2W columns (rows 2W apart),
 *                                  as yb_vae_unpatchify2_clamp; frame >= 4 * Hs * W
 *   yb_nhwc_to_nchw_f32_clamp_rows: x f32 [T * Hs * W, ldx] -> Cn channels x T frames x Hs rows x W columns (rows W apart),
 *                                  as yb_nhwc_to_nchw_f32_clamp; frame >= Hs * W */
int yb_vae_unpatchify2_clamp_rows(const void* y, long long ldy, void* out, long long plane, long long frame, int T, int Hs, int W,
                                  void* stream);
int yb_nhwc_to_nchw_f32_clamp_rows(const void* x, long long ldx, void* out, long long plane, long long frame, int T, int Hs,
                                   int W, int Cn, float lo, float hi, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* YUME_B200_VAE_ROWS_H_ */
