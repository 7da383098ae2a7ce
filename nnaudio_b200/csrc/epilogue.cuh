// Output-format epilogue shared by the SIMT and tensor-core framed kernels.
// Mirrors the element-wise tails of the reference forward() bodies:
//   STFT   stft.py:299-316     CQT1992v2  cqt.py:752-780
//   CQT2010v2 cqt.py:1112-1139 Mel/Gammatone power  mel.py:186
#pragma once

#include "common.cuh"

namespace nnab {

struct EpiParams {
  const float* scale;  // per-bin factor or nullptr
  float scale_all;
  int fmt;
  float eps;
  float power;
  float* out;
  int64_t T;
  int out_bins;
  int bin_offset;
  int F;
  const FbEntry* fb_table;  // FMT_FBANK
  const FbStep* fb_steps;   // FMT_FBANK, block-partial kernel
  int n_fb;
  DecimParams dec;          // FMT_DECIM
  float* raw;               // FMT_RAW: re plane; im plane at raw + raw_plane
  int64_t raw_plane;
  int64_t ola_pitch;        // FMT_OLA
  int ola_hop;
  int64_t planes_stride;    // FMT_PLANES (block-partial kernel): hi -> lo plane distance, elements
  int planes_pitch;         //   and elements per frame row; `out` is the plane base
};

__device__ __forceinline__ float epi_power(const EpiParams& e, float re, float im) {
  // |X| first, then ** power, like `stft(x, "Magnitude") ** self.power` (mel.py:186)
  float p = __fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im));
  if (e.eps != 0.f) p = __fadd_rn(p, e.eps);
  const float m = sqrtf(p);
  if (e.power == 2.0f) return __fmul_rn(m, m);
  if (e.power == 1.0f) return m;
  return powf(m, e.power);
}

// re/im are the final-signed contraction results for (clip b, bin f, frame t).
__device__ __forceinline__ void epi_store(const EpiParams& e, int64_t b, int f, int64_t t,
                                          float re, float im) {
  const int row = f + e.bin_offset;
  if (row < 0 || row >= e.out_bins) return;
  float s = e.scale_all;
  if (e.scale != nullptr) s *= __ldg(e.scale + f);
  re *= s;
  im *= s;
  const int64_t idx = ((int64_t)b * e.out_bins + row) * e.T + t;
  switch (e.fmt) {
    case NNAB_FMT_MAGNITUDE: {
      // pow(2) + pow(2) (+ eps) then sqrt, each step rounded like the reference
      float p = __fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im));
      if (e.eps != 0.f) p = __fadd_rn(p, e.eps);
      e.out[idx] = sqrtf(p);
    } break;
    case NNAB_FMT_COMPLEX: {
      reinterpret_cast<float2*>(e.out)[idx] = make_float2(re, im);
    } break;
    case NNAB_FMT_PHASE_ANGLE: {
      e.out[idx] = atan2f(im + 0.0f, re);
    } break;
    case NNAB_FMT_PHASE_UNIT: {
      const float ang = atan2f(im, re);
      float sn, cs;
      sincosf(ang, &sn, &cs);
      reinterpret_cast<float2*>(e.out)[idx] = make_float2(cs, sn);
    } break;
    default: {  // FMT_POWER
      float p = __fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im));
      if (e.eps != 0.f) p = __fadd_rn(p, e.eps);
      const float m = sqrtf(p);
      float v;
      if (e.power == 2.0f) v = __fmul_rn(m, m);
      else if (e.power == 1.0f) v = m;
      else v = powf(m, e.power);
      e.out[idx] = v;
    } break;
  }
}

// Compile-time-format variant for the tensor-core kernels: keeps the 32x unrolled
// accumulator read-out loop small enough to stay in the instruction cache.
//   FMT: 0..3 = NNAB_FMT_*, 4 = FMT_POWER, 9 = FMT_REALPAIR.  `dst` already points at element
//   (b, bin_offset, t) of the output (float2 elements for the 2-channel formats).
template <int FMT>
__device__ __forceinline__ void epi_store_fmt(const EpiParams& e, float* dst, int f, float re,
                                              float im) {
  const int row = f + e.bin_offset;
  if (row < 0 || row >= e.out_bins) return;
  float s = e.scale_all;
  if (e.scale != nullptr) s *= __ldg(e.scale + f);
  re *= s;
  im *= s;
  const int64_t off = (int64_t)f * e.T;
  if constexpr (FMT == NNAB_FMT_MAGNITUDE) {
    float p = __fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im));
    if (e.eps != 0.f) p = __fadd_rn(p, e.eps);
    dst[off] = sqrtf(p);
  } else if constexpr (FMT == NNAB_FMT_COMPLEX) {
    reinterpret_cast<float2*>(dst)[off] = make_float2(re, im);
  } else if constexpr (FMT == NNAB_FMT_PHASE_ANGLE) {
    dst[off] = atan2f(im + 0.0f, re);
  } else if constexpr (FMT == NNAB_FMT_PHASE_UNIT) {
    const float ang = atan2f(im, re);
    float sn, cs;
    sincosf(ang, &sn, &cs);
    reinterpret_cast<float2*>(dst)[off] = make_float2(cs, sn);
  } else if constexpr (FMT == 9) {
    // two real rows per complex column pair (real GEMMs on the complex kernel: dense filterbanks)
    dst[off] = re;
    if (row + e.F < e.out_bins) dst[off + (int64_t)e.F * e.T] = im;
  } else {
    float p = __fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im));
    if (e.eps != 0.f) p = __fadd_rn(p, e.eps);
    const float m = sqrtf(p);
    float v;
    if (e.power == 2.0f) v = __fmul_rn(m, m);
    else if (e.power == 1.0f) v = m;
    else v = powf(m, e.power);
    dst[off] = v;
  }
}

// running banded-filterbank sums of one bin stream (ascending or descending bins)
struct MelRun {
  int cj0 = -1, cj1 = -1;
  float a0 = 0.f, a1 = 0.f;
  __device__ __forceinline__ void add(const EpiParams& e, float* mel, bool valid, int bin, float pw) {
    const int4 raw = __ldg(reinterpret_cast<const int4*>(e.fb_table) + bin);
    if (raw.x != cj0) {
      if (raw.x == cj1) {
        const int tj = cj0; cj0 = cj1; cj1 = tj;
        const float ta = a0; a0 = a1; a1 = ta;
      } else {
        if (cj0 >= 0 && valid) atomicAdd(mel + (int64_t)cj0 * e.T, a0);
        cj0 = raw.x; a0 = 0.f;
      }
    }
    if (raw.y != cj1) {
      if (cj1 >= 0 && valid) atomicAdd(mel + (int64_t)cj1 * e.T, a1);
      cj1 = raw.y; a1 = 0.f;
    }
    a0 = fmaf(__int_as_float(raw.z), pw, a0);
    a1 = fmaf(__int_as_float(raw.w), pw, a1);
  }
  __device__ __forceinline__ void flush(const EpiParams& e, float* mel, bool valid) {
    if (cj0 >= 0 && valid) atomicAdd(mel + (int64_t)cj0 * e.T, a0);
    if (cj1 >= 0 && valid) atomicAdd(mel + (int64_t)cj1 * e.T, a1);
  }
};

}  // namespace nnab
