// Per-channel energy normalisation (PCEN, DESIGN.md §3.11): one forward kernel for the offline, training and
// streamed calls, one backward kernel (reverse-time scan) and the fixed-order reduction of its parameter partials.
//
// Every row (b, c) of a (B, C, T) spectrogram is a first-order recurrence in time,
//   M[t] = (1 - s) M[t-1] + s E[t]      (M[-1] = E[0], or the carried state of a primed stream slot)
// evaluated by ONE thread per row, frame by frame, with one fixed expression: chunked and whole-clip calls
// therefore agree bit for bit.  The block stages tiles of E through shared memory so that global loads and stores
// run along t (coalesced) while the 32 threads of the first warp own the 32 rows of the block; the compression
//   P[t] = bias^r expm1(r log1p(u / bias)),  u = E[t] (eps + M[t])^-gain
// has no dependence chain and runs on every thread of the block once the tile's M is known.
#include "common.cuh"

namespace nnab {

namespace {

constexpr int kRows = 32;      // rows per block: the lanes of the scanning warp
constexpr int kTile = 64;      // frames per shared-memory tile
constexpr int kThreads = 256;  // forward loads, stores and compression: 8 tile entries per thread
constexpr int kPer = kRows * kTile / kThreads;
constexpr int kBwdThreads = 128;  // the backward kernel: 16 entries per thread, whose partials stay in registers
constexpr int kBwdPer = kRows * kTile / kBwdThreads;

__device__ __forceinline__ int64_t min64(int64_t a, int64_t b) { return a < b ? a : b; }
__device__ __forceinline__ int64_t max64(int64_t a, int64_t b) { return a > b ? a : b; }

struct RowParams {
  float s, gain, bias, power;
};

__device__ __forceinline__ RowParams row_params(const PcenArgs& a, int64_t c) {
  const int64_t i = a.param_stride ? c : 0;
  return RowParams{a.s[i], a.gain[i], a.bias[i], a.power[i]};
}

// the smoother's update: the one expression every call evaluates
__device__ __forceinline__ float smooth(float oms, float s, float m, float e) {
  return __fmaf_rn(oms, m, __fmul_rn(s, e));
}

// (eps + M)^-gain as exp2(-gain log2(eps + M)): a few ulp, a fraction of powf's instructions
__device__ __forceinline__ float inv_gain(float me, float gain) { return exp2f(-gain * log2f(me)); }

// u = E (eps + M)^-gain
__device__ __forceinline__ float gained(float e, float m, float gain, float eps) {
  return e * inv_gain(eps + m, gain);
}

// P = bias^r expm1(r log1p(u / bias)): no cancellation when u << bias
__device__ __forceinline__ float compress(float u, float bias, float power, float bias_r) {
  return bias_r * expm1f(power * log1pf(u / bias));
}

__global__ void __launch_bounds__(kThreads) pcen_forward_kernel(const float* __restrict__ E, int64_t rows, int C,
                                                                int64_t T, PcenArgs a, float* __restrict__ P,
                                                                float* __restrict__ M_out, PcenStream st) {
  __shared__ float sE[kRows][kTile + 1];
  __shared__ float sM[kRows][kTile + 1];
  __shared__ float sGain[kRows], sBias[kRows], sPow[kRows], sBiasR[kRows];
  __shared__ int64_t sN[kRows];
  const int tid = threadIdx.x;
  const int64_t row0 = (int64_t)blockIdx.x * kRows;
  const int nrows = (int)min64(kRows, rows - row0);

  // the scanning lanes: per-row parameters, frame count and initial state
  float s = 0.f, oms = 0.f, m = 0.f;
  bool carried = false;
  int64_t sidx = -1;
  if (tid < kRows) {
    int64_t n = 0;
    if (tid < nrows) {
      const int64_t row = row0 + tid, b = row / C, c = row - b * C;
      const RowParams p = row_params(a, c);
      s = p.s;
      oms = 1.f - p.s;
      sGain[tid] = p.gain;
      sBias[tid] = p.bias;
      sPow[tid] = p.power;
      sBiasR[tid] = powf(p.bias, p.power);
      n = T;
      if (st.counts != nullptr) n = min64(max64(st.counts[b], 0), T);
      if (st.state != nullptr) {
        const int64_t slot = st.row_slot != nullptr ? (int64_t)st.row_slot[b] : b;
        if (slot >= 0 && slot < st.slots) {
          sidx = slot * C + c;
          carried = st.primed[sidx] != 0;
          if (carried) m = st.state[sidx];
        } else {
          n = 0;  // a row mapped outside the slots computes nothing
        }
      }
    }
    sN[tid] = n;
  }

  const float* Eb = E + row0 * T;
  float pre[kPer];
  auto load = [&](int64_t t0) {
    const int64_t tw = min64(kTile, T - t0);
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int i = tid + j * kThreads, r = i / kTile, k = i % kTile;
      pre[j] = (r < nrows && k < tw) ? Eb[(int64_t)r * T + t0 + k] : 0.f;
    }
  };
  if (T > 0) load(0);
  for (int64_t t0 = 0; t0 < T; t0 += kTile) {
    const int tw = (int)min64(kTile, T - t0);
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int i = tid + j * kThreads;
      sE[i / kTile][i % kTile] = pre[j];
    }
    __syncthreads();
    if (t0 + kTile < T) load(t0 + kTile);  // in flight while this tile is scanned and stored
    if (tid < kRows) {
      const int kend = (int)min64(max64(sN[tid] - t0, 0), tw);
      if (t0 == 0 && kend > 0 && !carried) m = sE[tid][0];  // M[-1] = E[0]: the smoother starts settled
#pragma unroll 8
      for (int k = 0; k < kend; ++k) {
        m = smooth(oms, s, m, sE[tid][k]);
        sM[tid][k] = m;
      }
    }
    __syncthreads();
#pragma unroll 4
    for (int j = 0; j < kPer; ++j) {
      const int i = tid + j * kThreads, r = i / kTile, k = i % kTile;
      if (r < nrows && k < tw) {
        const int64_t o = (row0 + r) * T + t0 + k;
        float out = 0.f;  // frames past a row's count are exact zeros
        if (t0 + k < sN[r]) out = compress(gained(sE[r][k], sM[r][k], sGain[r], a.eps), sBias[r], sPow[r], sBiasR[r]);
        P[o] = out;
        if (M_out != nullptr) M_out[o] = sM[r][k];
      }
    }
    __syncthreads();
  }
  if (tid < nrows && sidx >= 0 && sN[tid] > 0) {
    st.state[sidx] = m;
    st.primed[sidx] = 1;
  }
}

// Reverse-time adjoint.  For each tile, last to first: the compression's derivatives in parallel (dE's direct
// term, the local g_M, the gain / bias / power partials, the last three accumulated per thread in a fixed
// assignment), then the scanning lane of each row runs
//   G[t] = g_M[t] + (1 - s) G[t+1],  dE[t] += s G[t],  ds += G[t] (E[t] - M[t-1])
// with dE[0] += (1 - s) G[0] for the M[-1] = E[0] start.  Per-row partials go to `partial` (4, rows).
__global__ void __launch_bounds__(kBwdThreads) pcen_backward_kernel(const float* __restrict__ E,
                                                                 const float* __restrict__ M,
                                                                 const float* __restrict__ gP, int64_t rows, int C,
                                                                 int64_t T, PcenArgs a, float* __restrict__ dE,
                                                                 float* __restrict__ partial) {
  __shared__ float sE[kRows][kTile + 1];
  __shared__ float sM[kRows][kTile + 1];  // sM[r][k + 1] = M[t0 + k], sM[r][0] = M[t0 - 1]
  __shared__ float sG[kRows][kTile + 1];
  __shared__ float sD[kRows][kTile + 1];
  __shared__ float sGain[kRows], sBias[kRows], sPow[kRows], sBiasR[kRows], sBiasR1[kRows], sLogBias[kRows];
  const int tid = threadIdx.x;
  const int64_t row0 = (int64_t)blockIdx.x * kRows;
  const int nrows = (int)min64(kRows, rows - row0);

  float s = 0.f, oms = 0.f;
  if (tid < kRows && tid < nrows) {
    const int64_t row = row0 + tid, c = row % C;
    const RowParams p = row_params(a, c);
    s = p.s;
    oms = 1.f - p.s;
    sGain[tid] = p.gain;
    sBias[tid] = p.bias;
    sPow[tid] = p.power;
    sBiasR[tid] = powf(p.bias, p.power);
    sBiasR1[tid] = powf(p.bias, p.power - 1.f);
    sLogBias[tid] = logf(p.bias);
  }
  // entry j of this thread is always row tid / kTile + j kBwdThreads / kTile, frame tid % kTile of a tile: its
  // sums of the gain, bias and power derivatives stay in registers across tiles
  float acc_g[kBwdPer], acc_b[kBwdPer], acc_p[kBwdPer];
#pragma unroll
  for (int j = 0; j < kBwdPer; ++j) acc_g[j] = acc_b[j] = acc_p[j] = 0.f;
  float G = 0.f, ds = 0.f;
  const int64_t n_tiles = (T + kTile - 1) / kTile;
  for (int64_t ti = n_tiles - 1; ti >= 0; --ti) {
    const int64_t t0 = ti * kTile;
    const int tw = (int)min64(kTile, T - t0);
#pragma unroll
    for (int j = 0; j < kBwdPer; ++j) {
      const int i = tid + j * kBwdThreads, r = i / kTile, k = i % kTile;
      float e = 0.f, mm = 0.f, g = 0.f;
      if (r < nrows && k < tw) {
        const int64_t o = (row0 + r) * T + t0 + k;
        e = E[o];
        mm = M[o];
        g = gP[o];
      }
      sE[r][k] = e;
      sM[r][k + 1] = mm;
      sG[r][k] = g;
    }
    if (tid < nrows) {
      const int64_t o = (row0 + tid) * T;
      sM[tid][0] = t0 > 0 ? M[o + t0 - 1] : E[o];
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kBwdPer; ++j) {
      const int i = tid + j * kBwdThreads, r = i / kTile, k = i % kTile;
      if (r < nrows && k < tw) {
        const float e = sE[r][k], me = a.eps + sM[r][k + 1], g = sG[r][k];
        const float gain = sGain[r], bias = sBias[r], pw = sPow[r];
        const float scale = inv_gain(me, gain), u = e * scale;
        const float l = log1pf(u / bias), w = pw * l;
        const float gu = g * pw * sBiasR1[r] * expf((pw - 1.f) * l);  // dP/du = r (bias + u)^(r-1)
        sD[r][k] = gu * scale;                                          // dE, direct term
        sG[r][k] = -gain * gu * u / me;                                 // dP/dM through u
        acc_g[j] -= gu * u * logf(me);
        acc_p[j] += g * sBiasR[r] * (sLogBias[r] * expm1f(w) + expf(w) * l);
        acc_b[j] += g * pw * sBiasR1[r] * expm1f((pw - 1.f) * l);
      }
    }
    __syncthreads();
    if (tid < nrows) {
      for (int k = tw - 1; k >= 0; --k) {
        G = __fmaf_rn(oms, G, sG[tid][k]);
        ds = __fmaf_rn(G, sE[tid][k] - sM[tid][k], ds);
        float d = __fmaf_rn(s, G, sD[tid][k]);
        if (t0 + k == 0) d = __fmaf_rn(oms, G, d);  // M[-1] = E[0]
        sD[tid][k] = d;
      }
    }
    __syncthreads();
    if (dE != nullptr) {
#pragma unroll
      for (int j = 0; j < kBwdPer; ++j) {
        const int i = tid + j * kBwdThreads, r = i / kTile, k = i % kTile;
        if (r < nrows && k < tw) dE[(row0 + r) * T + t0 + k] = sD[r][k];
      }
    }
    __syncthreads();
  }
  if (partial == nullptr) return;
  // per-row sums of the per-thread partials, in frame-column order
#pragma unroll
  for (int j = 0; j < kBwdPer; ++j) {
    const int i = tid + j * kBwdThreads, r = i / kTile, k = i % kTile;
    sE[r][k] = acc_g[j];
    sG[r][k] = acc_b[j];
    sD[r][k] = acc_p[j];
  }
  __syncthreads();
  if (tid < nrows) {
    float sg = 0.f, sb = 0.f, sp = 0.f;
    for (int k = 0; k < kTile; ++k) {
      sg += sE[tid][k];
      sb += sG[tid][k];
      sp += sD[tid][k];
    }
    const int64_t row = row0 + tid;
    partial[row] = ds;
    partial[rows + row] = sg;
    partial[2 * rows + row] = sb;
    partial[3 * rows + row] = sp;
  }
}

// grad_params[q * n_out + c] = the sum of partial q over the rows of channel c (per-channel parameters: rows
// b * C + c for every b) or over every row (scalar parameters).  Fixed order: strided per-thread sums, then a
// shared-memory tree.
constexpr int kReduceThreads = 256;
__global__ void __launch_bounds__(kReduceThreads) pcen_param_reduce_kernel(const float* __restrict__ partial,
                                                                           int64_t rows, int C, int per_channel,
                                                                           float* __restrict__ grad_params) {
  __shared__ float red[kReduceThreads];
  const int q = blockIdx.y, c = blockIdx.x, n_out = gridDim.x;
  const float* p = partial + q * rows + (per_channel ? c : 0);
  const int64_t n = per_channel ? rows / C : rows, stride = per_channel ? C : 1;
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += kReduceThreads) acc += p[i * stride];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int h = kReduceThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) grad_params[(int64_t)q * n_out + c] = red[0];
}

__global__ void pcen_reset_kernel(uint8_t* primed, const uint8_t* __restrict__ mask, int64_t n, int C) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && (mask == nullptr || mask[i / C] != 0)) primed[i] = 0;
}

}  // namespace

int64_t pcen_blocks(int64_t rows) { return (rows + kRows - 1) / kRows; }

int pcen_forward(const float* E, int64_t B, int C, int64_t T, const PcenArgs& a, float* P, float* M_out,
                 const PcenStream& st, cudaStream_t stream) {
  const int64_t rows = B * C;
  pcen_forward_kernel<<<(unsigned)pcen_blocks(rows), kThreads, 0, stream>>>(E, rows, C, T, a, P, M_out, st);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

int pcen_backward(const float* E, const float* M, const float* gP, int64_t B, int C, int64_t T, const PcenArgs& a,
                  float* dE, float* grad_params, float* partial, cudaStream_t stream) {
  const int64_t rows = B * C;
  pcen_backward_kernel<<<(unsigned)pcen_blocks(rows), kBwdThreads, 0, stream>>>(
      E, M, gP, rows, C, T, a, dE, grad_params != nullptr ? partial : nullptr);
  NNAB_LAUNCH_CHECK();
  if (grad_params == nullptr) return NNAB_OK;
  const int n_out = a.param_stride ? C : 1;
  pcen_param_reduce_kernel<<<dim3((unsigned)n_out, 4), kReduceThreads, 0, stream>>>(partial, rows, C,
                                                                                     a.param_stride, grad_params);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

int pcen_reset(uint8_t* primed, const uint8_t* mask, int64_t slots, int C, cudaStream_t stream) {
  const int64_t n = slots * C;
  pcen_reset_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(primed, mask, n, C);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

}  // namespace nnab
