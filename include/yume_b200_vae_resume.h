/* yume_b200_vae_resume.h — C ABI of the frame comparison behind the Wan VAE engines' `resume=True` sessions in libyume_b200.so
 * (conventions as include/yume_b200.h: device pointers, `stream` a cudaStream_t as void*, no allocation, no synchronisation,
 * capture-safe launches, 0 or a negative YB_ERR_* code).
 *
 * A resuming engine keeps a copy of the input of its last call. The next call runs only its new latent frames when the new
 * input starts with the kept one bit for bit; the encoder can also resume where the kept input's trailing run of all-zero
 * frames began. Both facts come from one read-only pass over the two inputs, which may be several GB each. */
#ifndef YUME_B200_VAE_RESUME_H_
#define YUME_B200_VAE_RESUME_H_

#include "yume_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* kept [C, t_kept, frame_elems] and x [C, t, frame_elems], both dense and frame-major within each channel plane, elements of
 * elem_bytes (1, 2, 4 or 8) bytes. Writes two int32 into result (device memory):
 *   result[0]  the first frame f < min(t_kept, t) at which kept and x differ in any bit of any channel; min(t_kept, t) when
 *              none does. The comparison is bitwise: -0.0 differs from +0.0, NaN payloads count.
 *   result[1]  where x's trailing run of all-zero frames begins (every bit of every channel 0): one past x's last frame with a
 *              set bit, 0 when x is all zero, t when its last frame is not zero.
 * t_kept may be 0 (kept may then be null). Reads kept and x once, writes nothing else; result is overwritten, not accumulated
 * into. The widest of 16, 8, 4, 2 or 1-byte loads that divides both pointers and the frame's bytes is used. */
int yb_vae_frame_match(const void* kept, int t_kept, const void* x, int t, int C, long long frame_elems, int elem_bytes,
                       int* result, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* YUME_B200_VAE_RESUME_H_ */
