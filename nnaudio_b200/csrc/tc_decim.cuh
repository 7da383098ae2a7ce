// FIR-decimator epilogue shared by the tensor-core kernels (tc_kernels.cu FMT_DECIM, tct_kernels.cu
// fir_tc_kernel): a thread holds 2*half consecutive outputs of one clip in its accumulator row and writes
// them as the NEXT pyramid level -- bf16 hi/lo planes in the layout that level's kernels read
// (utils.py:73-124 conv1d(stride=2, padding=127); cqt.py:1065-1068 reflect padding per level).
#pragma once

#include <cuda_bf16.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace nnab {

__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// trow: accumulator-tile address of this warp's 32 rows (tc_ptx.cuh); tl: frame index inside clip b.
// [c_lo, c_hi): the accumulator columns (= outputs of the frame) this warp handles (c_hi < 0: all 2*half).
__device__ __forceinline__ void epilogue_decim(const DecimParams& d, uint32_t trow, int64_t b,
                                               int64_t tl, bool valid, int half, int c_lo = 0,
                                               int c_hi = -1) {
        // ---- FIR decimator stage: this thread holds outputs n0 .. n0 + 2*half - 1 of clip b ----
        const int64_t n0 = tl * (2 * half);
        __nv_bfloat16* pc = reinterpret_cast<__nv_bfloat16*>(d.pc);
        __nv_bfloat16* pf = reinterpret_cast<__nv_bfloat16*>(d.pf);
        if (c_hi < 0) c_hi = 2 * half;
#pragma unroll 1
        for (int c0 = c_lo; c0 < c_hi; c0 += 8) {
          uint32_t v[8];
          acc_ld8(trow + (uint32_t)c0, v);  // re half = outputs 0..half-1, im half = the rest
          const int64_t n = n0 + c0;
          if (valid && n < d.len_out) {
            __align__(16) __nv_bfloat16 hi[8];
            __align__(16) __nv_bfloat16 lo[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) split_bf16(__uint_as_float(v[e]), hi[e], lo[e]);
            const bool full = (n + 8 <= d.len_out);
            if (pf != nullptr) {
              __nv_bfloat16* q = pf + b * d.pf_pitch + 128 + n;
              if (full) {
                *reinterpret_cast<uint4*>(q) = *reinterpret_cast<const uint4*>(hi);
                *reinterpret_cast<uint4*>(q + d.pf_plane) = *reinterpret_cast<const uint4*>(lo);
              } else {
                for (int e = 0; e < 8 && n + e < d.len_out; ++e) { q[e] = hi[e]; q[d.pf_plane + e] = lo[e]; }
              }
            }
            if (pc != nullptr) {
              __nv_bfloat16* q = pc + b * d.pc_pitch + d.pc_off + n;
              if (full) {
                *reinterpret_cast<uint4*>(q) = *reinterpret_cast<const uint4*>(hi);
                *reinterpret_cast<uint4*>(q + d.pc_plane) = *reinterpret_cast<const uint4*>(lo);
              } else {
                for (int e = 0; e < 8 && n + e < d.len_out; ++e) { q[e] = hi[e]; q[d.pc_plane + e] = lo[e]; }
              }
              // nn.ReflectionPad1d margins of the next level: mirror samples 1..off and
              // len-1-off..len-2 (cqt.py:1065-1068 pads each level's own signal)
              if (d.pc_reflect && (n <= d.pc_off || n + 8 >= d.len_out - 1 - d.pc_off)) {
                __nv_bfloat16* base = pc + b * d.pc_pitch + d.pc_off;
                for (int e = 0; e < 8; ++e) {
                  const int64_t m = n + e;
                  if (m >= d.len_out) break;
                  if (m >= 1 && m <= d.pc_off) { base[-m] = hi[e]; base[d.pc_plane - m] = lo[e]; }
                  if (m >= d.len_out - 1 - d.pc_off && m <= d.len_out - 2) {
                    const int64_t r = 2 * (d.len_out - 1) - m;
                    base[r] = hi[e]; base[d.pc_plane + r] = lo[e];
                  }
                }
              }
            }
            if (d.y32 != nullptr) {
              float* q = d.y32 + b * d.y32_pitch + n;
              for (int e = 0; e < 8 && n + e < d.len_out; ++e) q[e] = __uint_as_float(v[e]);
            }
          }
        }
}

}  // namespace nnab
