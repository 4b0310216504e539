// yb_host.h — host-side helpers shared by the C-ABI translation units: error codes, TMA tensor-map
// encoding through the driver entry point (no link-time dependency on libcuda), launch checks.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cuda.h>
#include <cuda_runtime.h>

#include "../../include/yume_b200.h"

namespace yb {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<PFN_encodeTiled>(p);
    (void)cudaGetLastError();
  }
  return fn;
}

// 2D bf16 tensor map: global view [rows, cols] with row stride `ld` elements, box {box_cols, box_rows},
// 128-byte swizzle, out-of-bounds elements are filled with zeros.
inline int make_tmap_bf16_2d(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                             uint32_t box_rows, uint32_t box_cols) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return YB_ERR_NO_DRIVER;
  if ((reinterpret_cast<uintptr_t>(base) & 0xF) || ((ld * 2) & 0xF)) return YB_ERR_ALIGNMENT;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? YB_OK : YB_ERR_TENSORMAP;
}

// 3D bf16 tensor map: [chunks, rows, cols] with row stride `ld` and chunk stride `chunk_ld` (elements),
// box {box_cols, box_rows, 1}. Used for a K-split A operand: logical column k = chunk * cols + c.
inline int make_tmap_bf16_3d(CUtensorMap* tm, const void* base, uint64_t chunks, uint64_t rows, uint64_t cols,
                             uint64_t ld, uint64_t chunk_ld, uint32_t box_rows, uint32_t box_cols) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return YB_ERR_NO_DRIVER;
  if ((reinterpret_cast<uintptr_t>(base) & 0xF) || ((ld * 2) & 0xF) || ((chunk_ld * 2) & 0xF)) return YB_ERR_ALIGNMENT;
  cuuint64_t gdim[3] = {cols, rows, chunks};
  cuuint64_t gstride[2] = {ld * 2, chunk_ld * 2};
  cuuint32_t box[3] = {box_cols, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? YB_OK : YB_ERR_TENSORMAP;
}

// 4D bf16 tensor map over a dense channels-last volume [T, H, W, C], box {bc, bw, bh, bt} (conv3d A operand).
inline int make_tmap_bf16_4d(CUtensorMap* tm, const void* base, uint64_t T, uint64_t H, uint64_t W, uint64_t C,
                             uint32_t bt, uint32_t bh, uint32_t bw, uint32_t bc, uint32_t st = 1, uint32_t sh = 1,
                             uint32_t sw = 1) {
  // st/sh/sw > 1: the map samples every s-th voxel of that axis (elementStrides); a box of b OUTPUT voxels spans b*s input voxels
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return YB_ERR_NO_DRIVER;
  if ((reinterpret_cast<uintptr_t>(base) & 0xF) || ((C * 2) & 0xF)) return YB_ERR_ALIGNMENT;
  cuuint64_t gdim[4] = {C, W, H, T};
  cuuint64_t gstride[3] = {C * 2, W * C * 2, H * W * C * 2};
  cuuint32_t box[4] = {bc, bw * sw, bh * sh, bt * st};
  cuuint32_t estr[4] = {1, sw, sh, st};
  if (box[1] > 256 || box[2] > 256 || box[3] > 256) return YB_ERR_SHAPE;
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? YB_OK : YB_ERR_TENSORMAP;
}

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    fprintf(stderr, "yume_b200: %s launch failed: %s\n", what, cudaGetErrorString(e));
    return YB_ERR_LAUNCH;
  }
  return YB_OK;
}

constexpr int kMaxDevices = 64;
inline int current_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
  return dev;
}

// SM count of the CURRENT device (cached per device: a process may drive several GPUs)
inline int sm_count() {
  static int n[kMaxDevices] = {0};
  const int dev = current_device();
  if (n[dev] == 0) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    n[dev] = v > 0 ? v : 132;   // H100 SXM
  }
  return n[dev];
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device property of a kernel: set it once per (kernel, device).
// `done` is the caller's static bool[kMaxDevices] for that kernel instance.
template <class Kern>
inline int ensure_dynamic_smem(Kern kern, int bytes, bool* done, const char* what) {
  const int dev = current_device();
  if (done[dev]) return YB_OK;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) {
    fprintf(stderr, "yume_b200: %s: cudaFuncSetAttribute(MaxDynamicSharedMemorySize=%d) failed: %s\n", what, bytes,
            cudaGetErrorString(e));
    (void)cudaGetLastError();
    return YB_ERR_LAUNCH;
  }
  done[dev] = true;
  return YB_OK;
}

}  // namespace yb
