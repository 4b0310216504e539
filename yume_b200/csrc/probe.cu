// probe.cu — single-tile self-test of the wgmma building blocks the GEMM and attention kernels rely on:
// TMA 128B-swizzled tiles, wgmma shared-memory descriptors for K-major and MN-major operands, and the
// A-operand-in-registers form. Test infrastructure only (tests/test_gpu_parity.py); never on the product path.
#include "yb_host.h"
#include "yb_ptx.cuh"

namespace yb {

// 256 threads: warpgroup w computes rows [64w, 64w + 64) of D = A (128 x 128) * B (128 x 128, per mode)
__global__ void __launch_bounds__(256, 1)
umma_probe_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __nv_bfloat16* __restrict__ Ag, float* __restrict__ D, int mode) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // modes 0..2: A = 2 slabs x 16 KB. modes >= 3 (row-shifted A, shift = mode - 2 rows): A = 2 slabs x 17 KB holding a
  // 136-row TMA box; the MMA reads rows [shift, shift + 128) by moving the descriptor start address by shift * 128 B.
  const int shift = mode >= 3 ? mode - 2 : 0;
  const uint32_t a_slab = shift ? 17408u : 16384u;
  uint8_t* sA = smem;
  uint8_t* sB = smem + 36864;   // 2 slabs x 16 KB
  uint64_t* bar_load = reinterpret_cast<uint64_t*>(smem + 69632);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int q4 = lane >> 2, c2 = 2 * (lane & 3);
  const int ra = wg * 64 + (warp & 3) * 16 + q4, rb = ra + 8;   // fragment rows of this thread

  if (threadIdx.x == 0) {
    mbar_init(bar_load, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(bar_load, 32768 + 2 * a_slab);
    tma_load_2d(sA, &tmA, bar_load, 0, 0);
    tma_load_2d(sA + a_slab, &tmA, bar_load, 64, 0);
    tma_load_2d(sB, &tmB, bar_load, 0, 0);
    tma_load_2d(sB + 16384, &tmB, bar_load, 64, 0);
  }
  mbar_wait(bar_load, 0);
  float d[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.f;
  const uint32_t a0 = smem_u32(sA) + wg * 64 * 128, b0 = smem_u32(sB);
  wgmma_fence();
  if (mode == 0 || mode >= 3) {
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint32_t off = (kk >> 2) * 16384 + (kk & 3) * 32;
      const uint32_t offa = (kk >> 2) * a_slab + (kk & 3) * 32 + shift * 128;
      wgmma_ss_acc64<0>(d, make_smem_desc_sw128(a0 + offa, 16, 1024), make_smem_desc_sw128(b0 + off, 16, 1024), kk != 0);
    }
  } else if (mode == 1) {
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint32_t offa = (kk >> 2) * 16384 + (kk & 3) * 32;
      wgmma_ss_acc64<1>(d, make_smem_desc_sw128(a0 + offa, 16, 1024), make_smem_desc_sw128(b0 + kk * 2048, 16384, 1024), kk != 0);
    }
  } else {
    // A from registers: the m64k16 fragment of k-step kk is (row a | row b) x (columns 16kk + c2, +1 | 16kk + 8 + c2, +1)
    const uint32_t* arow_a = reinterpret_cast<const uint32_t*>(Ag + ra * 128);
    const uint32_t* arow_b = reinterpret_cast<const uint32_t*>(Ag + rb * 128);
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint32_t a[4] = {arow_a[(16 * kk + c2) / 2], arow_b[(16 * kk + c2) / 2], arow_a[(16 * kk + 8 + c2) / 2],
                             arow_b[(16 * kk + 8 + c2) / 2]};
      wgmma_rs_n128_tb(d, a, make_smem_desc_sw128(b0 + kk * 2048, 16384, 1024), kk != 0);
    }
  }
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(d);
#pragma unroll
  for (int g = 0; g < 16; ++g) {
    *reinterpret_cast<float2*>(D + ra * 128 + 8 * g + c2) = make_float2(d[4 * g], d[4 * g + 1]);
    *reinterpret_cast<float2*>(D + rb * 128 + 8 * g + c2) = make_float2(d[4 * g + 2], d[4 * g + 3]);
  }
}

}  // namespace yb

extern "C" int yb_umma_probe(const void* A, const void* B, void* D, int mode, void* stream_) {
  using namespace yb;
  if (!A || !B || !D || mode < 0 || mode > 10) return YB_ERR_ARG;
  CUtensorMap tmA, tmB;
  int rc = make_tmap_bf16_2d(&tmA, A, 128, 128, 128, mode >= 3 ? 136 : 128, 64);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmB, B, 128, 128, 128, 128, 64);
  if (rc) return rc;
  const int smem = 69632 + 1024 + 64;
  static bool attr_set[kMaxDevices] = {false};
  if (int rc2 = ensure_dynamic_smem(umma_probe_kernel, smem, attr_set, "umma_probe")) return rc2;
  umma_probe_kernel<<<1, 256, smem, reinterpret_cast<cudaStream_t>(stream_)>>>(
      tmA, tmB, static_cast<const __nv_bfloat16*>(A), static_cast<float*>(D), mode);
  return check_launch("umma_probe");
}
