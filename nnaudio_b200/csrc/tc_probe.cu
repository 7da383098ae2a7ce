// Hardware probe (test infrastructure, not on any product path): does a K-major SWIZZLE_128B wgmma
// shared-memory descriptor address an operand that starts at an arbitrary ROW of a TMA-written
// block (start address = block + r * 128 B), and what must the descriptor's base-offset field
// (bits 49..51) hold for it?  The tall-A kernels (tct_kernels.cu) read overlapping (Toeplitz) A tiles
// in place from one tall block and rely on the answer "any row, base offset 0".
//   out[v][r][128][32] = A[r .. r+128) x B^T  for row offsets r = 0..15 and
//   v = 0: base_offset = 0        v = 1: base_offset = r & 7
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "tc_ptx.cuh"
#include "tc_host.cuh"

namespace nnab {

constexpr int PROBE_ROWS = 144, PROBE_N = 32, PROBE_R = 16;

__global__ void __launch_bounds__(128, 1)
probe_rowoffset_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                       float* __restrict__ out) {
  const uint32_t base = acc_tile_base();
  const uint32_t a_s = base;                           // 144 rows x 128 B = 18 KB
  const uint32_t b_s = base + 20 * 1024;               // 32 rows x 128 B
  const uint32_t bar = base + 28 * 1024;
  const int t = threadIdx.x;
  if (t == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (t == 0) {
    mbar_expect_tx(bar, PROBE_ROWS * 128 + PROBE_N * 128);
    tma_load_3d(a_s, &tm_a, bar, 0, 0, 0);
    tma_load_3d(b_s, &tm_b, bar, 0, 0, 0);
  }
  mbar_wait(bar, 0);
  const uint32_t row_in_half = (t >> 5) * 16 + ((t & 31) >> 2), col = (t & 3) * 2;
  for (int v = 0; v < 2; ++v) {
    for (int r = 0; r < PROBE_R; ++r) {
      for (int h = 0; h < 2; ++h) {  // the two m64 halves of the 128 rows
        float d[PROBE_N / 2];
#pragma unroll
        for (int i = 0; i < PROBE_N / 2; ++i) d[i] = 0.f;
        const uint32_t hi = wg_desc_hi() | (v == 1 ? (uint32_t)(r & 7) << 17 : 0u);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t da = desc64(wg_desc_lo(a_s + (uint32_t)(r + 64 * h) * 128u + (uint32_t)k * 32u), hi);
          const uint64_t db = desc64(wg_desc_lo(b_s + (uint32_t)k * 32u), wg_desc_hi());
          Wgmma<PROBE_N>::mma(d, da, db, k > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait_all();
        float* o = out + (((size_t)v * PROBE_R + r) * 128 + 64 * h + row_in_half) * PROBE_N + col;
#pragma unroll
        for (int j = 0; j < PROBE_N / 8; ++j) {
          o[8 * j] = d[4 * j];
          o[8 * j + 1] = d[4 * j + 1];
          o[8 * PROBE_N + 8 * j] = d[4 * j + 2];
          o[8 * PROBE_N + 8 * j + 1] = d[4 * j + 3];
        }
      }
    }
  }
}

// a: (144, 64) bf16, b: (32, 64) bf16, out: (2, 16, 128, 32) fp32 -- all device pointers
int tc_probe_rowoffset(const void* a, const void* b, float* out, cudaStream_t stream) {
  CUtensorMap ma, mb;
  int rc = encode_3d(&ma, const_cast<void*>(a), 64, PROBE_ROWS, 1, 128, (uint64_t)PROBE_ROWS * 128, 64,
                     PROBE_ROWS, 64);
  if (rc) return rc;
  rc = encode_3d(&mb, const_cast<void*>(b), 64, PROBE_N, 1, 128, (uint64_t)PROBE_N * 128, 64, PROBE_N, 64);
  if (rc) return rc;
  const int smem = 32 * 1024;
  probe_rowoffset_kernel<<<1, 128, smem, stream>>>(ma, mb, out);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

}  // namespace nnab

extern "C" __attribute__((visibility("default"))) int nnab_probe_rowoffset(const void* a, const void* b,
                                                                         float* out, void* stream) {
  if (a == nullptr || b == nullptr || out == nullptr) return NNAB_EINVAL;
  return nnab::tc_probe_rowoffset(a, b, out, (cudaStream_t)stream);
}
