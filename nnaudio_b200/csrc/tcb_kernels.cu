// Block-partial ("sliding") STFT on wgmma for sm_90a — the default kernel of the STFT family
// (STFT / MelSpectrogram / MFCC / Gammatonegram with a periodic Hann window and hop = n_fft / R,
// R = 2 or 4: the reference's defaults, stft.py:177-178).
//
// The dense path contracts every frame with the windowed n_fft-point basis (features/stft.py:290-293:
// conv1d(x, wsin/wcos, stride=hop)).  Consecutive frames share R-1 of their R hop-sized blocks, so
// here the contraction runs ONCE per block against the UN-windowed basis:
//
//   Z_g[k]  = sum_{n < hop} xpad[g*hop + n] exp(-2 pi i k n / N)                    K = hop, not N
//   hann[m] = 1/2 - 1/4 e^{+i theta m} - 1/4 e^{-i theta m}    (theta = 2 pi / N)   3 taps along k
//   X_t[k]  = sum_{j<R} c_k^j V_j(Z_{t+j})[k],   c_k = exp(-2 pi i k / R)
//   V_j(Z)[k] = 1/2 Z[k] - 1/4 w^j Z[k-1] - 1/4 w^-j Z[k+1],   w = exp(2 pi i / R)
//
// (tools/block_dft_emulation.py is the executable spec; exact in exact arithmetic.)  R times fewer
// MMA flops than the dense form, the A operand is a plain (blocks x hop) matrix, and the epilogue
// does the R-block frame sum with warp shuffles and the 3-tap bin filter in registers, in that order:
//   S_t[k] = sum_{j<R} c_k^j Z_{t+j}[k],   X_t[k] = 1/2 S_t[k] - 1/4 (S_t[k-1] + S_t[k+1])
// (the same sum, since c_k w = c_{k-1}; tools/block_epilogue_emulation.py).
//
// GEMM view: M = block rows g of the whole batch (the split-signal planes of tc_kernels.cu viewed
// as a (rows x hop) matrix), K = hop, N = 2 * (F + 2) columns (re | im of bins -1 .. F: the two
// extra bins are the k-1 / k+1 neighbours of the edge bins).
//
// Tiling (same pipeline roles as framed_tc_kernel, tc_ptx.cuh):
//   * N tile = nb packed bins, re rows then im rows (MMA N = 2 nb); consecutive tiles overlap by
//     2 bins, a tile emits nb - 2 output bins.
//   * M: each epilogue warp owns one 32-row quarter of the accumulator tile = 32 consecutive block
//     rows and emits 33 - R frames; the 4 quarters of a tile are loaded as four 32-row TMA boxes whose
//     row origins are 33 - R apart, so no frame needs a row of another warp (no exchange, no barrier).
//     4 * (33 - R) frames per tile (116 of 128 rows for R = 4).
//   * fp32 parity: x*w = xhi*whi + xlo*whi + xhi*wlo on bf16 tensor cores, fp32 accumulation.  A bf16
//     waveform has xlo = 0: that kernel instance (PASSES = 2) skips the xlo*whi pass and the A lo plane.
//
// Four phases (PH = 4, whenever hop % 128 == 0): only hop of the N samples of Z_g are non-zero, so the N-point
// block DFT is split by decimation in time.  With M = N / 4 and the polyphase rows x_q[m] = x[g hop + 4 m + q]
// (m < hop / 4, stored in that order by the pre-pass, TC_SPLIT_POLY4):
//
//   Y_q(k') = sum_m x_q[m] e^{-2 pi i k' m / M},   k' = -1 .. M/2 + 1      K = hop / 4, ONE basis for all q
//   T_q = e^{-2 pi i k' q / N} Y_q,   A0 = T0 + T2, A1 = T0 - T2, B0 = T1 + T3, B1 = T1 - T3
//   Z[k'] = A0 + B0   Z[M + k'] = A1 - i B1   Z[M - k'] = conj(A1 + i B1)   Z[2M - k'] = conj(A0 - B0)
//
// (tools/block_poly_emulation.py is the executable spec.)  A quarter of the MMA work and of the operand bytes.
// The rows of an M tile's A operand are the 4 phases of the same 32 block rows, laid out so that one thread's
// accumulators hold all four phases of one (block row, packed bin): each warpgroup runs both m64 slabs h = 0, 1
// (slab row 16 w + 8 p + i = phase 2 h + p of block row 8 w + i) against its half of the N columns, and the packed
// basis keeps each bin's re and im rows next to each other (tcb_poly_tile).  The butterfly then runs on the
// registers, and its four families go into the accumulator tile as quarter f = family f (f1, f3 column-reversed
// so that every family runs over ascending bins, common.cuh block_family_span); the epilogue above runs on each
// quarter with its family's bin origin and bin range.  33 - R frames per tile.
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "epilogue.cuh"
#include "tc_ptx.cuh"
#include "tc_host.cuh"
#include "tc_decim.cuh"

namespace nnab {

constexpr int TCB_BK = 32;          // K block: one 64-byte swizzled row per operand row
constexpr int TCB_MAX_STAGES = 4;

struct TcbParams {
  int num_m_tiles;   // 128-row tiles along M (4 * (33 - R) frames each; 33 - R with four phases)
  int num_n_tiles;
  int nb;            // packed bins per N tile (MMA N = 2 nb)
  int kb_n;          // K / TCB_BK (K = hop, or hop / 4 with four phases)
  int stages;        // ring depth, TcbSmem::stages(nb)
  int c_split;       // warp part 0 of a quarter owns the 8-column chunks [0, c_split), part 1 the rest
  int fam_M;         // four phases: M = n_fft / 4 (family bins, block_family_span); 0 with one phase
  const float2* twiddle;  // four phases: [q - 1][p] = e^{-2 pi i (p - 1) q / N}, q = 1 .. 3
  int tw_rows;
  int64_t nv, t_slots, T;
  EpiParams epi;
};

// Dynamic shared memory: [1024-byte alignment slack][accumulator tile][stage ring][barriers].  The
// accumulator tile has its own space, so the producer refills the ring while the epilogue reads the tile.
// PASSES = 3: the split product xlo*whi + xhi*wlo + xhi*whi, a stage holds both A planes.  PASSES = 2 (a
// bf16 waveform, xlo == 0): xhi*wlo + xhi*whi, a stage holds the A hi plane only, so the ring may be deeper.
struct TcbSmem {
  static constexpr uint32_t A_BYTES = TC_BM * TCB_BK * 2;  // one plane, 128 rows
  static constexpr uint32_t LIMIT = 227 * 1024;            // opt-in dynamic shared memory per block
  // the ring's full / empty barriers, the fused filterbank's hand-over sums (4 quarters x 32 rows x 2), then the
  // accumulator tile's full / empty barriers of framed_tcb_ws_kernel
  static constexpr uint32_t HANDOVER_OFF = 16 * TCB_MAX_STAGES;
  static constexpr uint32_t ACC_BARS_OFF = HANDOVER_OFF + 4 * 32 * 8;
  static constexpr uint32_t BAR_BYTES = ACC_BARS_OFF + 16;
  // 128 fp32 rows of 2 nb columns, rounded up to 32 columns (acc_tile)
  __host__ __device__ static uint32_t acc_bytes(int nb) { return TC_BM * (uint32_t)((2 * nb + 31) / 32) * 128u; }
  // one (plane, part) box of the basis: nb rows; a multiple of 512 B, so every operand starts on an atom
  __host__ __device__ static uint32_t part_bytes(int nb) { return (uint32_t)nb * TCB_BK * 2; }
  // A planes per stage: 2 (hi, lo) with three passes, 1 (hi) with two
  __host__ __device__ static constexpr uint32_t a_planes(int passes) { return passes == 3 ? 2u : 1u; }
  __host__ __device__ static uint32_t stage_bytes(int nb, int passes) {
    return a_planes(passes) * A_BYTES + 4 * part_bytes(nb);
  }
  // `extra`: bytes a kernel keeps behind the barriers (framed_tcb_ws_kernel's fused-filterbank action slices)
  static int stages(int nb, int passes, uint32_t extra = 0) {
    const int s = (int)((LIMIT - 1024 - BAR_BYTES - extra - acc_bytes(nb)) / stage_bytes(nb, passes));
    return s < TCB_MAX_STAGES ? s : TCB_MAX_STAGES;
  }
  static uint32_t total(int nb, int passes, uint32_t extra = 0) {
    return 1024 + acc_bytes(nb) + stages(nb, passes, extra) * stage_bytes(nb, passes) + BAR_BYTES + extra;
  }
};

// rows of one (plane, part) slab of the packed block basis
static int block_choose_nb(int F) {
  int best = 32, best_cost = 1 << 30;
  for (int nb = 128; nb >= 32; nb -= 8) {
    const int tiles = (F + nb - 3) / (nb - 2);
    const int cost = tiles * (nb + 6);  // + a little per-tile overhead: prefer fewer, wider tiles on ties
    if (cost < best_cost) { best_cost = cost; best = nb; }
  }
  return best;
}
static int block_n_tiles(int F, int nb) { return (F + nb - 3) / (nb - 2); }
// rows of one (plane, part) slab: bins -1 .. F plus zero rows so that the last tile of ANY nb <= 128
// stays inside the slab (the launch picks nb, e.g. wider tiles for the fused filterbank)
static int block_p_rows(int F) { return round_up_i(F + 2 + 128, 8); }

// The four-phase form: K = hop / 4 in K blocks of 32, and the packed "bins" are k' = 0 .. M/2 (F' = M/2 + 1).
static bool block_poly4(int hop) { return hop % 128 == 0; }
// packed bins of the basis (F of the one-phase form, F' with four phases) and its K
static int block_basis_F(int n_fft, int hop) { return block_poly4(hop) ? n_fft / 8 + 1 : n_fft / 2 + 1; }
static int block_basis_K(int hop) { return block_poly4(hop) ? hop / 4 : hop; }
// byte offset of the four-phase twiddle table behind the basis slabs
static size_t block_twiddle_offset(int n_fft, int hop) {
  const size_t slabs = (size_t)4 * block_p_rows(block_basis_F(n_fft, hop)) * block_basis_K(hop) * sizeof(__nv_bfloat16);
  return (slabs + 255) / 256 * 256;
}

size_t tc_packed_block_bytes(int n_fft, int hop) {
  if (!tc_block_shape_ok(n_fft, hop)) return 0;
  size_t n = block_twiddle_offset(n_fft, hop);
  if (block_poly4(hop)) n += (size_t)3 * block_p_rows(block_basis_F(n_fft, hop)) * sizeof(float2);
  return n + 256;
}

void tc_block_tile_geometry(int n_fft, int hop, int* nb, int* n_tiles, int* phases) {
  const int F = block_basis_F(n_fft, hop);
  *nb = block_choose_nb(F);
  *n_tiles = block_n_tiles(F, *nb);
  *phases = block_poly4(hop) ? 4 : 1;
}

bool tc_block_shape_ok(int n_fft, int hop) {
  if (hop <= 0 || n_fft % hop != 0) return false;
  const int R = n_fft / hop;
  return (R == 2 || R == 4) && hop % 64 == 0 && n_fft >= 128 && n_fft <= 32768;
}

// packed[plane hi|lo][part re|im][p][n]: bin k = p - 1, sample n < hop:
//   re row:  cos(2 pi k n / N)      im row: -sin(2 pi k n / N)     (so re + i im = e^{-i theta k n})
// Four phases: the same rows of the M-point DFT over hop / 4 samples (n_fft = M, hop = hop / 4, F = F'), stored
// interleaved (`pairs`) as packed[plane][p][part re|im][n], so that a tile's re and im rows of bin p are MMA
// columns 2 p and 2 p + 1 and either half of the tile's columns is one contiguous run of rows.  Same bytes.
__global__ void __launch_bounds__(256) pack_block_basis_kernel(int n_fft, int hop, int F, int p_rows, bool pairs,
                                                               __nv_bfloat16* __restrict__ packed) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int k8 = hop / 8;
  if (idx >= (int64_t)p_rows * k8) return;
  const int p = (int)(idx / k8);
  const int n0 = (int)(idx % k8) * 8;
  const int k = p - 1;
  __align__(16) __nv_bfloat16 rh[8], rl[8], ih[8], il[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    float c = 0.f, s = 0.f;
    if (p < F + 2) {
      const int n = n0 + e;
      long long m = ((long long)k * n) % n_fft;
      if (m < 0) m += n_fft;
      double sd, cd;
      sincospi(2.0 * (double)m / (double)n_fft, &sd, &cd);
      c = (float)cd;
      s = (float)(-sd);
    }
    rh[e] = __float2bfloat16_rn(c);
    rl[e] = __float2bfloat16_rn(c - __bfloat162float(rh[e]));
    ih[e] = __float2bfloat16_rn(s);
    il[e] = __float2bfloat16_rn(s - __bfloat162float(ih[e]));
  }
  const int64_t slab = (int64_t)p_rows * hop;
  const int64_t o = (int64_t)(pairs ? 2 * p : p) * hop + n0;  // re row of bin p in the hi plane
  const int64_t im = pairs ? hop : slab;                      // its im row
  *reinterpret_cast<uint4*>(packed + o) = *reinterpret_cast<const uint4*>(rh);
  *reinterpret_cast<uint4*>(packed + o + im) = *reinterpret_cast<const uint4*>(ih);
  *reinterpret_cast<uint4*>(packed + 2 * slab + o) = *reinterpret_cast<const uint4*>(rl);
  *reinterpret_cast<uint4*>(packed + 2 * slab + o + im) = *reinterpret_cast<const uint4*>(il);
}

// four phases: tw[q - 1][p] = e^{-2 pi i k q / N}, k = p - 1, q = 1 .. 3 (fp32, from float64)
__global__ void __launch_bounds__(256) pack_block_twiddle_kernel(int n_fft, int p_rows, float2* __restrict__ tw) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= 3 * p_rows) return;
  const int q = idx / p_rows + 1, p = idx - (q - 1) * p_rows;
  long long m = ((long long)(p - 1) * q) % n_fft;
  if (m < 0) m += n_fft;
  double sd, cd;
  sincospi(2.0 * (double)m / (double)n_fft, &sd, &cd);
  tw[idx] = make_float2((float)cd, (float)(-sd));
}

int tc_pack_basis_block(int n_fft, int hop, void* packed, cudaStream_t stream) {
  if (!tc_block_shape_ok(n_fft, hop) || packed == nullptr) return NNAB_EINVAL;
  const bool poly = block_poly4(hop);
  const int F = block_basis_F(n_fft, hop), K = block_basis_K(hop);
  const int p_rows = block_p_rows(F);
  const int64_t threads = (int64_t)p_rows * (K / 8);
  pack_block_basis_kernel<<<(unsigned)ceil_div64(threads, 256), 256, 0, stream>>>(
      poly ? n_fft / 4 : n_fft, K, F, p_rows, poly, (__nv_bfloat16*)packed);
  NNAB_LAUNCH_CHECK();
  if (poly) {
    pack_block_twiddle_kernel<<<(unsigned)ceil_div64(3 * p_rows, 256), 256, 0, stream>>>(
        n_fft, p_rows, reinterpret_cast<float2*>((char*)packed + block_twiddle_offset(n_fft, hop)));
    NNAB_LAUNCH_CHECK();
  }
  mark_packed(packed, PACK_BLOCK, n_fft, hop);
  return NNAB_OK;
}

// ---------------------------------------------------------------------------
// epilogue: one warp = one 32-row quarter of the accumulator tile (32 consecutive block rows) x a range
// of 8-column chunks.  The arithmetic of a chunk is straight-line code, so the 8 columns' dependency chains
// (shuffles and twiddles -> 3-tap filter -> magnitude) interleave: with one or two warps per scheduler the
// epilogue is latency-bound, not issue-bound.
// ---------------------------------------------------------------------------
__device__ __forceinline__ float sqrt_approx(float x) {
  float r;
  asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));  // <= 1 ulp-ish: far below the 1e-4 bar
  return r;
}

// FMT 5 fast path: static action list and the default power 2 without eps; anything else (other powers,
// trainable eps, no action list) takes the rolled MelRun path
__device__ __forceinline__ bool fb_fast_path(const EpiParams& e) {
  return e.fb_steps != nullptr && e.power == 2.0f && e.eps == 0.f;
}

// |X|^2 from 2X: (2X)^2 times the exact 1/4, the same float as rounding |X|^2 itself (outside subnormals)
__device__ __forceinline__ float power_of_2x(float yr, float yi) {
  return __fmul_rn(0.25f, __fadd_rn(__fmul_rn(yr, yr), __fmul_rn(yi, yi)));
}

// fire-and-forget fp32 add, predicated (no branch: the chunk body stays one basic block)
__device__ __forceinline__ void red_add_if(float* addr, float v, bool on) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %2, 0;\n\t"
      "@p red.global.add.f32 [%0], %1;\n\t}"
      ::"l"(addr), "f"(v), "r"((int)on)
      : "memory");
}

// One quarter of the tile holds a run of packed columns over ascending bins: output o (column o + 1) is bin
// k_tile0 + o, and the outputs with bins in [klo, khi) are this quarter's to emit.  FMT_PLANES writes chunk c
// at plane column col0 + 8 c.
//
// Four phases, fused filterbank: the two warps of a quarter (parts 0, 1, cut at chunk c_split) hand over the
// sums of the filters open at the cut.  Part 1 keeps the first flush of each slot, which belongs to the filter
// part 0 ends with, and passes it through shared memory (`handover`, named barrier 2 + quarter); part 0 adds it
// to its own final sum before its one atomic add.  So a filter gets one partial sum per (family, tile).
//
// Fused filterbank actions: without STAGED they are read from fb_steps with __ldg, a chunk ahead of its
// arithmetic; with STAGED, `acts` is the warp's copy in shared memory of fb_steps entries k_tile0 + 8 c_begin - 3
// .. k_tile0 + 8 c_end - 3 (tcb_stage_actions), read where they are used.
template <int FMT, int R, int PH, bool STAGED = false>
__device__ __forceinline__ void epilogue_tile_block(const TcbParams& p, uint32_t trow, int64_t g, int lane,
                                                    int k_tile0, int klo, int khi, int64_t col0, int c_begin,
                                                    int c_end, int part, int quarter, uint32_t handover,
                                                    const int4* acts) {
  const int nb = p.nb;
  const int64_t b = g / p.t_slots;
  const int64_t t = g - b * p.t_slots;  // frame index inside the clip = index of its first block
  const bool valid = (lane < 33 - R) && (g < p.nv) && (t < p.T);
  constexpr int CH = (FMT == NNAB_FMT_COMPLEX) ? 2 : 1;
  float* dst = nullptr;
  float* mel = nullptr;
  if constexpr (FMT == 5) mel = p.epi.out + ((int64_t)b * p.epi.n_fb) * p.epi.T + t;
  else if constexpr (FMT != 9) dst = p.epi.out + (((int64_t)b * p.epi.out_bins + p.epi.bin_offset) * p.epi.T + t) * CH;
  MelRun run;
  const bool fast_fb = (FMT == 5) && fb_fast_path(p.epi);
  float ma = 0.f, mb = 0.f;  // FMT 5, static action list: the two running filter sums
  int mca = -1, mcb = -1;    //   and the filters they currently belong to
  constexpr bool HANDOVER = FMT == 5 && PH == 4;
  bool first_a = false, first_b = false;  // part 1: the next flush of the slot is the filter open at the cut
  float head_a = 0.f, head_b = 0.f;
  if constexpr (HANDOVER) {
    const int kq = k_tile0 + 8 * c_begin - 3;  // the bin before this part's first
    if (fast_fb && part == 1 && kq >= 0) {
      const int w = STAGED ? acts[0].w : __ldg(reinterpret_cast<const int4*>(p.epi.fb_steps) + kq).w;
      first_a = (short)(w & 0xffff) >= 0;
      first_b = (short)((unsigned)w >> 16) >= 0;
    }
  }

  // twiddles c_k of the 4 residues the unrolled loop meets: packed column 8c + e is bin
  // k = k_tile0 + 8c + e - 1, so k mod 4 = (k_tile0 + 3 + e) mod 4 (8c drops out).
  float cr[4], ci[4], c2[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = (k_tile0 + 3 + i) & 3;
    if constexpr (R == 4) {  // c = (-i)^k
      cr[i] = (m == 0) ? 1.f : ((m == 2) ? -1.f : 0.f);
      ci[i] = (m == 3) ? 1.f : ((m == 1) ? -1.f : 0.f);
    } else {
      cr[i] = 0.f; ci[i] = 0.f;
    }
    c2[i] = (m & 1) ? -1.f : 1.f;  // R = 4: c^2 = (-1)^k;  R = 2: c = (-1)^k
  }
  // S_t = sum_{j<R} c^j Z_{t+j} of one packed column, row t = lane (the rows past 32 - R read garbage that no
  // valid lane uses).  R = 4 as pair sums: Q_t = Z_t + c Z_{t+1}, S_t = Q_t + c^2 Q_{t+2}.
  auto frame_sum = [&](float zr, float zi, int i, float& s_r, float& s_i) {
    const float z1r = __shfl_down_sync(0xffffffffu, zr, 1), z1i = __shfl_down_sync(0xffffffffu, zi, 1);
    if constexpr (R == 4) {
      const float qr = fmaf(cr[i], z1r, fmaf(-ci[i], z1i, zr)), qi = fmaf(cr[i], z1i, fmaf(ci[i], z1r, zi));
      const float q2r = __shfl_down_sync(0xffffffffu, qr, 2), q2i = __shfl_down_sync(0xffffffffu, qi, 2);
      s_r = fmaf(c2[i], q2r, qr);
      s_i = fmaf(c2[i], q2i, qi);
    } else {
      s_r = fmaf(c2[i], z1r, zr);
      s_i = fmaf(c2[i], z1i, zi);
    }
  };

  float wr[10], wi[10];  // S of packed columns 8c-2 .. 8c+7 of this row (re, im)
  wr[8] = wr[9] = wi[8] = wi[9] = 0.f;
  if (c_begin > 0) {  // a column range that starts inside the tile: seed the two carried columns
    uint32_t re[8], im[8];
    acc_ld8(trow + (uint32_t)(8 * (c_begin - 1)), re);
    acc_ld8(trow + (uint32_t)(nb + 8 * (c_begin - 1)), im);
    frame_sum(__uint_as_float(re[6]), __uint_as_float(im[6]), 2, wr[8], wi[8]);
    frame_sum(__uint_as_float(re[7]), __uint_as_float(im[7]), 3, wr[9], wi[9]);
  }
#pragma unroll 1
  for (int c = c_begin; c < c_end; ++c) {
    wr[0] = wr[8]; wr[1] = wr[9]; wi[0] = wi[8]; wi[1] = wi[9];
    int4 st[8];  // FMT 5 from fb_steps: this chunk's filterbank actions, requested before the accumulator loads
    if constexpr (FMT == 5) {
      if (!STAGED && fast_fb) {
        const int kq = k_tile0 + 8 * c - 2;
#pragma unroll
        for (int e = 0; e < 8; ++e)
          st[e] = __ldg(reinterpret_cast<const int4*>(p.epi.fb_steps) + (kq + e < 0 ? 0 : kq + e));
      }
    }
    {
      uint32_t re[8], im[8];
      acc_ld8(trow + (uint32_t)(8 * c), re);
      acc_ld8(trow + (uint32_t)(nb + 8 * c), im);
#pragma unroll
      for (int e = 0; e < 8; ++e) frame_sum(__uint_as_float(re[e]), __uint_as_float(im[e]), e & 3, wr[e + 2], wi[e + 2]);
    }
    // the Hann window on the frame sums: X[k] = 1/2 S[k] - 1/4 (S[k-1] + S[k+1]).  xr / xi hold 2 X; the exact
    // factor 1/2 is applied by the format tails (1/4 on the power, power_of_2x).
    float xr[8], xi[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      xr[e] = fmaf(-0.5f, wr[e] + wr[e + 2], wr[e + 1]);
      xi[e] = fmaf(-0.5f, wi[e] + wi[e + 2], wi[e + 1]);
    }
    const int k0 = k_tile0 + 8 * c - 2;          // bin of e = 0 (outputs -2, -1 of chunk 0 do not exist)
    const int e_lo = (c == 0) ? 2 : 0;
    auto own = [&](int e) { return e >= e_lo && k0 + e >= klo && k0 + e < khi; };
    if constexpr (FMT == NNAB_FMT_MAGNITUDE || FMT == NNAB_FMT_COMPLEX || FMT == 4) {
      float* q = dst + (int64_t)k0 * p.epi.T * CH;
      const int64_t step = p.epi.T * CH;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const bool ok = valid && own(e);
        if constexpr (FMT == NNAB_FMT_COMPLEX) {
          if (ok) *reinterpret_cast<float2*>(q) = make_float2(0.5f * xr[e], 0.5f * xi[e]);
        } else {
          float pw = power_of_2x(xr[e], xi[e]);
          if (p.epi.eps != 0.f) pw = __fadd_rn(pw, p.epi.eps);
          float v;
          if constexpr (FMT == NNAB_FMT_MAGNITUDE) {
            v = sqrt_approx(pw);
          } else {  // |X| ** power (mel.py:186); ** 2 is the power spectrum itself to 1 ulp
            v = (p.epi.power == 2.0f) ? pw
                : ((p.epi.power == 1.0f) ? sqrt_approx(pw) : powf(sqrt_approx(pw), p.epi.power));
          }
          if (ok) *q = v;
        }
        q += step;
      }
    } else if constexpr (FMT == 9) {
      // operand planes of the dense-filterbank GEMM (FMT_PLANES): frame (b, t) is row b * T + t, the 8
      // packed columns of chunk c of tile n (family f) sit at nb * (PH n + f) + 8 c (16-byte aligned: nb is a
      // multiple of 8), |X| ** power as bf16 hi / lo.  The two columns a tile repeats from its left neighbour,
      // the bins another family emits and the bins past F are written as zeros (the re-indexed bank has zero
      // rows there).
      __align__(16) __nv_bfloat16 hi[8];
      __align__(16) __nv_bfloat16 lo[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float pw = power_of_2x(xr[e], xi[e]);
        if (p.epi.eps != 0.f) pw = __fadd_rn(pw, p.epi.eps);
        float v = (p.epi.power == 2.0f) ? pw
                  : ((p.epi.power == 1.0f) ? sqrt_approx(pw) : powf(sqrt_approx(pw), p.epi.power));
        if (!own(e)) v = 0.f;
        split_bf16(v, hi[e], lo[e]);
      }
      if (valid) {
        __nv_bfloat16* q = reinterpret_cast<__nv_bfloat16*>(p.epi.out) +
                           (b * p.epi.T + t) * (int64_t)p.epi.planes_pitch + col0 + 8 * c;
        *reinterpret_cast<uint4*>(q) = *reinterpret_cast<const uint4*>(hi);
        *reinterpret_cast<uint4*>(q + p.epi.planes_stride) = *reinterpret_cast<const uint4*>(lo);
      }
    } else if constexpr (FMT == 5) {
      if (fast_fb) {
        // banded filterbank, static action list: two running sums per row.  Bins this quarter does not own
        // (the two columns of chunk 0 that belong to the previous tile, another family's bins, bins past F)
        // contribute with power 0.  power == 2 (the default, mel.py:186: |X| ** 2): the power spectrum itself.
        const int4* a = acts + 8 * (c - c_begin) + 1;  // (STAGED) the chunk's 8 actions
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float pw = own(e) ? power_of_2x(xr[e], xi[e]) : 0.f;
          const int z = STAGED ? a[e].z : st[e].z;
          // a filter ends at ~1 bin in 6 (and at the same bins for every row): one warp-uniform test
          // on the packed flush word keeps the address / predicate / RED code off the common path
          if (__any_sync(0xffffffffu, z != -1)) {
            const int fa = (int)(short)(z & 0xffff), fb = (int)(short)((unsigned)z >> 16);
            bool keep_a = false, keep_b = false;
            if constexpr (HANDOVER) {
              keep_a = first_a && fa >= 0;
              keep_b = first_b && fb >= 0;
              head_a = keep_a ? ma : head_a;
              head_b = keep_b ? mb : head_b;
              first_a = first_a && !keep_a;
              first_b = first_b && !keep_b;
            }
            red_add_if(mel + (int64_t)fa * p.epi.T, ma, fa >= 0 && valid && !keep_a);
            red_add_if(mel + (int64_t)fb * p.epi.T, mb, fb >= 0 && valid && !keep_b);
            ma = fa >= 0 ? 0.f : ma;
            mb = fb >= 0 ? 0.f : mb;
          }
          ma = fmaf(__int_as_float(STAGED ? a[e].x : st[e].x), pw, ma);
          mb = fmaf(__int_as_float(STAGED ? a[e].y : st[e].y), pw, mb);
        }
        const int cur = STAGED ? a[7].w : st[7].w;  // filters the two sums belong to after this chunk
        mca = (int)(short)(cur & 0xffff);
        mcb = (int)(short)((unsigned)cur >> 16);
      } else {
#pragma unroll 1
        for (int e = e_lo; e < 8; ++e) {
          const int k = k0 + e;
          if (k >= khi) break;  // warp-uniform
          if (k < klo) continue;
          float re = xr[0], im = xi[0];
#pragma unroll
          for (int j = 1; j < 8; ++j) { re = (e == j) ? xr[j] : re; im = (e == j) ? xi[j] : im; }
          run.add(p.epi, mel, valid, k, epi_power(p.epi, 0.5f * re, 0.5f * im));
        }
      }
    } else {
      // atan2f tail: rolled per bin (code size), after the straight-line part
#pragma unroll 1
      for (int e = e_lo; e < 8; ++e) {
        const int k = k0 + e;
        if (k >= khi) break;  // warp-uniform
        if (k < klo) continue;
        // dynamic index into xr/xi would spill: select with a short unrolled scan
        float re = xr[0], im = xi[0];
#pragma unroll
        for (int j = 1; j < 8; ++j) { re = (e == j) ? xr[j] : re; im = (e == j) ? xi[j] : im; }
        if (valid) epi_store_fmt<FMT>(p.epi, dst, k, 0.5f * re, 0.5f * im);
      }
    }
  }
  if constexpr (HANDOVER) {
    if (fast_fb) {
      const uint32_t slot = handover + (uint32_t)(quarter * 32 + lane) * 8u;
      if (part == 1) {
        if (first_a) { head_a = ma; mca = -1; }  // no flush in this part: its whole sum is the open filter's
        if (first_b) { head_b = mb; mcb = -1; }
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(slot), "f"(head_a), "f"(head_b) : "memory");
        asm volatile("bar.arrive %0, 64;" ::"r"(2 + quarter) : "memory");
      } else {
        asm volatile("bar.sync %0, 64;" ::"r"(2 + quarter) : "memory");
        float ha, hb;
        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(ha), "=f"(hb) : "r"(slot) : "memory");
        ma += ha;
        mb += hb;
      }
    }
  }
  if constexpr (FMT == 5) {
    red_add_if(mel + (int64_t)mca * p.epi.T, ma, mca >= 0 && valid);
    red_add_if(mel + (int64_t)mcb * p.epi.T, mb, mcb >= 0 && valid);
  }
  if constexpr (FMT == 5) run.flush(p.epi, mel, valid);
}

// Epilogue warps: all 8 consumer warps, 2 per 32-row quarter of the tile (column halves).  For the fused
// filterbank the two halves are also FB_EPI_PARTS, the range cuts fb_steps was built for.
constexpr int TCB_PARTS = 2;
static_assert(FB_EPI_PARTS == TCB_PARTS, "fused-filterbank column ranges follow the epilogue warps");

// The stage ring.  A stage holds A (hi, lo planes, or hi only with two passes; 128 rows each) and B (hi, lo
// planes of 2 nb rows each); its empty barrier counts the 8 consumer warps.
struct TcbRing {
  uint32_t base, stage_bytes, bars;
  int stages;
  __device__ uint32_t stage(int s) const { return base + (uint32_t)s * stage_bytes; }
  __device__ uint32_t full(int s) const { return bars + 8u * s; }
  __device__ uint32_t empty(int s) const { return bars + 8u * (TCB_MAX_STAGES + s); }
};

// One K block of tile (m_tile, n_tile) into ring stage `stage` (the stage's full barrier expects its bytes).
template <int R, int PASSES, int PH>
__device__ __forceinline__ void tcb_load_block(const CUtensorMap* tm_a, const CUtensorMap* tm_b, const TcbRing& ring,
                                               int stage, int m_tile, int n_tile, int kb, int nb) {
  using S = TcbSmem;
  constexpr int BK = TCB_BK;
  constexpr int FW = 33 - R;  // frames per warp quarter
  constexpr int TILE_ROWS = PH == 4 ? FW : 4 * FW;  // block rows an M tile advances
  const int m0 = m_tile * TILE_ROWS;
  const int n0 = n_tile * (nb - 2);
  const uint32_t sb = ring.stage(stage);
  const uint32_t full = ring.full(stage);
  mbar_expect_tx(full, ring.stage_bytes);
  const int k0 = kb * BK;
  const uint32_t b = sb + S::a_planes(PASSES) * S::A_BYTES;
  const uint32_t part_bytes = S::part_bytes(nb);
  if constexpr (PH == 4) {
    // tm_a is (k, block row, phase, plane): a 16-row box is phases 2 h, 2 h + 1 of block rows m0 + 8 w .. + 7,
    // slab h rows 16 w .. 16 w + 15 (tcb_poly_tile's row map)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const uint32_t dst = sb + (uint32_t)(64 * h + 16 * w) * BK * 2u;
        tma_load_4d(dst, tm_a, full, k0, m0 + 8 * w, 2 * h, 0);
        if constexpr (PASSES == 3) tma_load_4d(dst + S::A_BYTES, tm_a, full, k0, m0 + 8 * w, 2 * h, 1);
      }
    }
    // B: one box of 2 nb rows per plane (bins n0 .. n0 + nb - 1, re and im rows interleaved)
    tma_load_3d(b, tm_b, full, k0, 2 * n0, 0);
    tma_load_3d(b + 2 * part_bytes, tm_b, full, k0, 2 * n0, 1);
  } else {
#pragma unroll
    for (int q = 0; q < 4; ++q) {  // 32-row boxes, row origins FW apart
      tma_load_3d(sb + (uint32_t)q * 32u * BK * 2u, tm_a, full, k0, m0 + q * FW, 0);
      if constexpr (PASSES == 3)
        tma_load_3d(sb + S::A_BYTES + (uint32_t)q * 32u * BK * 2u, tm_a, full, k0, m0 + q * FW, 1);
    }
    // B rows [0, nb) = re part, [nb, 2 nb) = im part of each plane: accumulator columns of the N = 2 nb MMA
#pragma unroll
    for (int j = 0; j < 4; ++j) tma_load_3d(b + (uint32_t)j * part_bytes, tm_b, full, k0, n0, j);
  }
}

struct TcbNoRefill {
  __device__ void operator()(int) const {}
};

// One tile's K loop: SLABS m64 slabs of A (the first at byte a_off of a stage, the next 64 rows on) against N
// columns of B (from byte b_off of each B plane), accumulators acc[h N / 2 ..] for slab h.  One phase: one slab,
// this warpgroup's, at N = 2 nb; four phases: both slabs at N = nb (tcb_poly_tile).  Each K block is committed as
// one wgmma group; the stage of the PREVIOUS block is released once that group has retired, so one group is
// always in flight.  A width fixed at compile time keeps every in-flight wgmma off divergent paths (ptxas would
// serialise them).  `refill(kb)` runs after K block kb's release: the warp-specialised kernel refills the released stage
// from one MMA thread, a divergent path, so there (IN_FLIGHT = 0) each block's group retires before its stage is
// released.
template <int N, int PASSES, int SLABS, int IN_FLIGHT = 1, class Refill = TcbNoRefill>
__device__ __forceinline__ void tcb_mainloop(float* acc, const TcbRing& ring, int kb_n, uint32_t a_off,
                                             uint32_t b_off, uint32_t part_bytes, int lane, int& stage,
                                             uint32_t& phase, Refill refill = Refill()) {
  static_assert(IN_FLIGHT == 0 || IN_FLIGHT == 1, "at most one wgmma group in flight");
  using S = TcbSmem;
  int prev = 0;
  for (int kb = 0; kb < kb_n; ++kb) {
    mbar_wait(ring.full(stage), phase);
    const uint32_t sb = ring.stage(stage);
    const uint32_t b = sb + S::a_planes(PASSES) * S::A_BYTES + b_off;
    wgmma_fence();
#pragma unroll
    for (int h = 0; h < SLABS; ++h) {
      const uint32_t a = sb + a_off + (uint32_t)h * 64u * (TCB_BK * 2);
      if constexpr (PASSES == 3)
        wg_kblock_split3_n<N, TCB_BK>(acc + h * (N / 2), wg_desc_lo(a), wg_desc_lo(a + S::A_BYTES), wg_desc_lo(b),
                                      wg_desc_lo(b + 2 * part_bytes), kb != 0);
      else
        wg_kblock_split2_n<N, TCB_BK>(acc + h * (N / 2), wg_desc_lo(a), wg_desc_lo(b),
                                      wg_desc_lo(b + 2 * part_bytes), kb != 0);
    }
    wgmma_commit();
    wgmma_wait<IN_FLIGHT>();
    __syncwarp();
    if (IN_FLIGHT == 0 || kb > 0) {
      if (lane == 0) mbar_arrive(ring.empty(IN_FLIGHT == 0 ? stage : prev));
      refill(IN_FLIGHT == 0 ? kb : kb - 1);
    }
    prev = stage;
    if (++stage == ring.stages) { stage = 0; phase ^= 1u; }
  }
  if constexpr (IN_FLIGHT == 1) {
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(ring.empty(prev));
    refill(kb_n - 1);
  }
}

// Four phases: one tile at MMA width N = nb.  Each warpgroup runs both m64 slabs of the A tile against its half of
// the packed columns (bins wg nb / 2 .. + nb / 2 - 1, re and im interleaved), so with slab row 16 w + 8 p + i =
// phase 2 h + p of block row 8 w + i, thread `lane` of warp w holds, for its block row r = 8 w + lane / 4 and bins
// c = wg nb / 2 + 4 j + lane % 4:
//   Y_0 = acc[4 j], acc[4 j + 1]   Y_1 = acc[4 j + 2], acc[4 j + 3]   (slab 0: rows 16 w + lane / 4, + 8)
//   Y_2, Y_3 the same at acc[N / 2 + ..]                              (slab 1)
// (re, im of each).  The radix-4 butterfly runs on those registers, in place, and once `wait()` has returned the
// four families go into the accumulator tile: family f of bin c at row 32 f + r, column c (f0, f2) or nb - 1 - c
// (f1, f3), re at that column, im nb columns on.  The four threads of a quad write 4 consecutive columns of one
// row and a warp's eight quads 8 rows of distinct r & 7, so under acc_chunk_smem's row XOR every store is
// conflict-free.  Column c's twiddles are Y_q's factors e^{-2 pi i k' q / N}, k' = n_tile (nb - 2) + c - 1.
template <int N>
__device__ __forceinline__ void tcb_butterfly_regs(const TcbParams& p, float* acc, int n_tile, int wg, int lane) {
  const float2* __restrict__ tw = p.twiddle + n_tile * (N - 2) + wg * (N / 2) + (lane & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    float yr[4], yi[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int o = (q >> 1) * (N / 2) + 4 * j + 2 * (q & 1);
      yr[q] = acc[o];
      yi[q] = acc[o + 1];
    }
    float tr[4], ti[4];
    tr[0] = yr[0]; ti[0] = yi[0];
#pragma unroll
    for (int q = 1; q < 4; ++q) {
      const float2 w = __ldg(tw + (q - 1) * p.tw_rows + 4 * j);
      tr[q] = w.x * yr[q] - w.y * yi[q];
      ti[q] = w.x * yi[q] + w.y * yr[q];
    }
    const float a0r = tr[0] + tr[2], a0i = ti[0] + ti[2], a1r = tr[0] - tr[2], a1i = ti[0] - ti[2];
    const float b0r = tr[1] + tr[3], b0i = ti[1] + ti[3], b1r = tr[1] - tr[3], b1i = ti[1] - ti[3];
    float fr[4], fi[4];
    fr[0] = a0r + b0r;  fi[0] = a0i + b0i;     // Z[k']
    fr[1] = a1r - b1i;  fi[1] = -(a1i + b1r);  // Z[M - k'] = conj(A1 + i B1)
    fr[2] = a1r + b1i;  fi[2] = a1i - b1r;     // Z[M + k'] = A1 - i B1
    fr[3] = a0r - b0r;  fi[3] = b0i - a0i;     // Z[2M - k'] = conj(A0 - B0)
#pragma unroll
    for (int f = 0; f < 4; ++f) {  // family f where phase f was
      const int o = (f >> 1) * (N / 2) + 4 * j + 2 * (f & 1);
      acc[o] = fr[f];
      acc[o + 1] = fi[f];
    }
  }
}

// The accumulator tile is 2 N columns wide, so its row stride is a compile-time constant and the four families'
// rows of one thread differ by immediates; acc_chunk_smem's row XOR is the same for all of them (32 f + r = r mod 8).
template <int N>
__device__ __forceinline__ void tcb_store_families(const float* acc, int wg, int warp, int lane) {
  constexpr uint32_t STRIDE = (uint32_t)((2 * N + 31) / 32) * 128u;
  const uint32_t r = (uint32_t)(8 * (warp & 3) + (lane >> 2));
  const uint32_t row0 = acc_tile_base() + r * STRIDE;
  const uint32_t swz = (r & 7u) << 4;  // acc_chunk_smem: 16-byte chunk c at position c ^ (row & 7)
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const uint32_t c = (uint32_t)(wg * (N / 2) + 4 * j + (lane & 3));
#pragma unroll
    for (int f = 0; f < 4; ++f) {
      const int o = (f >> 1) * (N / 2) + 4 * j + 2 * (f & 1);
      const uint32_t col = (f & 1) ? (uint32_t)(N - 1) - c : c;
      const uint32_t at = row0 + 32u * f * STRIDE;
      asm volatile("st.shared.f32 [%0], %1;" ::"r"(at + ((4u * col) ^ swz)), "f"(acc[o]) : "memory");
      asm volatile("st.shared.f32 [%0], %1;" ::"r"(at + ((4u * (N + col)) ^ swz)), "f"(acc[o + 1]) : "memory");
    }
  }
}

template <int N, int PASSES, int IN_FLIGHT, class Wait, class Refill = TcbNoRefill>
__device__ __forceinline__ void tcb_poly_tile(const TcbParams& p, float* acc, const TcbRing& ring, int n_tile,
                                              int warp, int lane, int& stage, uint32_t& phase, Wait wait,
                                              Refill refill = Refill()) {
  const int wg = warp >> 2;
  const uint32_t part_bytes = TcbSmem::part_bytes(N);
  tcb_mainloop<N, PASSES, 2, IN_FLIGHT>(acc, ring, p.kb_n, 0u, (uint32_t)wg * part_bytes, part_bytes, lane, stage,
                                        phase, refill);
  tcb_butterfly_regs<N>(p, acc, n_tile, wg, lane);
  wait();
  tcb_store_families<N>(acc, wg, warp, lane);
}

// One warp's share of a tile's epilogue: 32-row quarter `quarter` (four phases: family `quarter`) and column
// part `part` of the accumulator tile.
template <int FMT, int R, int PH, bool STAGED = false>
__device__ __forceinline__ void tcb_epilogue(const TcbParams& p, uint32_t tile_addr, int m_tile, int n_tile,
                                             int quarter, int part, int lane, uint32_t handover,
                                             const int4* acts = nullptr) {
  constexpr int FW = 33 - R;  // frames per warp quarter
  constexpr int TILE_ROWS = PH == 4 ? FW : 4 * FW;  // block rows an M tile advances
  const int nb = p.nb;
  const int c_begin = part == 0 ? 0 : p.c_split, c_end = part == 0 ? p.c_split : nb / 8;
  const int64_t g = (int64_t)m_tile * TILE_ROWS + (PH == 4 ? 0 : quarter * FW) + lane;
  int k_tile0, klo, khi;
  block_family_span(n_tile, PH == 4 ? quarter : 0, nb, PH == 4 ? p.fam_M : 0, p.epi.F, &k_tile0, &klo, &khi);
  if (klo < k_tile0) klo = k_tile0;
  const int64_t col0 = (int64_t)nb * (PH * n_tile + (PH == 4 ? quarter : 0));
  epilogue_tile_block<FMT, R, PH, STAGED>(p, tile_addr + acc_row((uint32_t)quarter * 32u), g, lane, k_tile0, klo,
                                          khi, col0, c_begin, c_end, part, quarter, handover, acts);
}

// Four phases, fused filterbank: copy the fb_steps entries warp (quarter, part) of tile n_tile reads into its
// shared-memory slice `acts` (epilogue_tile_block, STAGED).  They do not depend on the accumulators, so the
// warp-specialised kernel loads them before it waits for the tile.  Negative bins read entry 0.
__device__ __forceinline__ void tcb_stage_actions(const TcbParams& p, int n_tile, int quarter, int part, int lane,
                                                  int4* acts) {
  if (!fb_fast_path(p.epi)) return;
  const int c_begin = part == 0 ? 0 : p.c_split, c_end = part == 0 ? p.c_split : p.nb / 8;
  int k_tile0, klo, khi;
  block_family_span(n_tile, quarter, p.nb, p.fam_M, p.epi.F, &k_tile0, &klo, &khi);
  const int base = k_tile0 + 8 * c_begin - 3;
  const int4* __restrict__ steps = reinterpret_cast<const int4*>(p.epi.fb_steps);
  __syncwarp();  // every lane is done with the previous tile's slice
  for (int i = lane; i <= 8 * (c_end - c_begin); i += 32) acts[i] = __ldg(steps + (base + i < 0 ? 0 : base + i));
  __syncwarp();
}

template <int FMT, int R, int PASSES, int PH>
__global__ void __launch_bounds__(TC_KERNEL_THREADS, 1)
framed_tcb_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                  const TcbParams p) {
  constexpr int BK = TCB_BK;
  static_assert(PH == 1 || PH == 4, "one or four phases");
  using S = TcbSmem;
  const int nb = p.nb;
  TcbRing ring;
  ring.base = acc_tile_base() + S::acc_bytes(nb);
  ring.stage_bytes = S::stage_bytes(nb, PASSES);
  ring.stages = p.stages;
  ring.bars = ring.base + (uint32_t)p.stages * ring.stage_bytes;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(ring.full(s), 1);
      mbar_init(ring.empty(s), 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int num_tiles = p.num_m_tiles * p.num_n_tiles;
  const uint32_t part_bytes = S::part_bytes(nb);

  if (warp == TC_PRODUCER_WARP) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      prefetch_tmap(&tm_a);
      prefetch_tmap(&tm_b);
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_tile = tile / p.num_n_tiles;
        const int n_tile = tile - m_tile * p.num_n_tiles;
        for (int kb = 0; kb < p.kb_n; ++kb) {
          mbar_wait(ring.empty(stage), phase ^ 1u);
          tcb_load_block<R, PASSES, PH>(&tm_a, &tm_b, ring, stage, m_tile, n_tile, kb, nb);
          if (++stage == p.stages) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  // ===================== consumers: wgmma, then the epilogue =====================
  const int wg = warp >> 2;
  const uint32_t a_off = (uint32_t)wg * 64u * (BK * 2);
  const uint32_t tile_addr = acc_tile(2 * nb);
  float acc[128];
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m_tile = tile / p.num_n_tiles;
    const int n_tile = tile - m_tile * p.num_n_tiles;
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    if constexpr (PH == 4) {
      // the butterfly on the registers; the families are stored once every warp is done reading the previous tile
      auto wait = [] { consumer_sync(); };
      switch (nb) {  // nb = 32 .. 128 in steps of 8
#define NNAB_TCB_CASE(N) \
  case N: tcb_poly_tile<N, PASSES, 1>(p, acc, ring, n_tile, warp, lane, stage, phase, wait); break;
        NNAB_TCB_CASE(32) NNAB_TCB_CASE(40) NNAB_TCB_CASE(48) NNAB_TCB_CASE(56) NNAB_TCB_CASE(64)
        NNAB_TCB_CASE(72) NNAB_TCB_CASE(80) NNAB_TCB_CASE(88) NNAB_TCB_CASE(96) NNAB_TCB_CASE(104)
        NNAB_TCB_CASE(112) NNAB_TCB_CASE(120) NNAB_TCB_CASE(128)
#undef NNAB_TCB_CASE
        default: break;
      }
    } else {
      switch (2 * nb) {  // nb = 32 .. 128 in steps of 8
#define NNAB_TCB_CASE(N) \
  case N: tcb_mainloop<N, PASSES, 1>(acc, ring, p.kb_n, a_off, 0u, part_bytes, lane, stage, phase); break;
        NNAB_TCB_CASE(64) NNAB_TCB_CASE(80) NNAB_TCB_CASE(96) NNAB_TCB_CASE(112) NNAB_TCB_CASE(128)
        NNAB_TCB_CASE(144) NNAB_TCB_CASE(160) NNAB_TCB_CASE(176) NNAB_TCB_CASE(192) NNAB_TCB_CASE(208)
        NNAB_TCB_CASE(224) NNAB_TCB_CASE(240) NNAB_TCB_CASE(256)
#undef NNAB_TCB_CASE
        default: break;
      }
      consumer_sync();  // every warp is done reading the previous tile
      acc_store<256>(tile_addr, acc, 2 * nb, wg * 64);
    }
    consumer_sync();
    // warp w: tile rows 32 (w & 3) .. + 31 (four phases: family w & 3), column part w >> 2
    tcb_epilogue<FMT, R, PH>(p, tile_addr, m_tile, n_tile, warp & 3, warp >> 2, lane, ring.bars + S::HANDOVER_OFF);
  }
}

// Four phases at nb <= TCB_WS_NB_MAX: the same tile schedule, ring, wgmma sequence and per-tile arithmetic as
// framed_tcb_kernel, with separate warps for separate roles, so a tile's MMAs run while the previous tile drains:
//   * warps 0-7 (two warpgroups): the K loop of tile i + 1 and the butterfly in registers while tile i is drained;
//     then, once the epilogue warps have released the accumulator tile (acc_empty), the family stores and acc_full.
//     Thread 0 also issues the TMA loads: after each release it waits until all 8 warps have released the stage
//     and refills it with the block `stages` ahead (across tile ends, so the next tile's first blocks land while
//     the MMA warps wait for acc_empty);
//   * warps 8-15: the epilogue, warp 8 + w in the place of consumer warp w of framed_tcb_kernel.
// 16 warps, because the register file is split over the four schedulers: 4 warps each get 128 registers, room for
// the 88 accumulators of two MMAs of width TCB_WS_NB_MAX (tcb_poly_tile).  A separate producer warp
// (17 warps) would cut every thread to 96, and ptxas does not raise the allocation inside setmaxnreg regions.
// There is one accumulator tile: two do not fit beside a stage at nb = 88 (2 x 96 KB + 38 KB > 227 KB), so a tile
// still takes store + epilogue; the MMAs and the butterfly are what is hidden.  With the fused filterbank the epilogue
// warps' fb_steps slices (TCB_WS_ACT_BYTES) sit behind the barriers: at nb = 88 the ring keeps its 3 stages, at
// nb = 80 (three passes) it has 3 instead of 4.
constexpr int TCB_WS_THREADS = 512;
constexpr int TCB_WS_NB_MAX = 88;
// fused filterbank: each epilogue warp's slice of fb_steps (tcb_stage_actions), 8 entries per chunk of its larger
// column part plus the one before, behind the barriers
constexpr int TCB_WS_ACTS = 8 * (TCB_WS_NB_MAX / 8 - TCB_WS_NB_MAX / 8 / TCB_PARTS) + 1;
constexpr uint32_t TCB_WS_ACT_BYTES = 8 * TCB_WS_ACTS * sizeof(int4);

template <int FMT, int R, int PASSES>
__global__ void __launch_bounds__(TCB_WS_THREADS, 1)
framed_tcb_ws_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                     const TcbParams p) {
  using S = TcbSmem;
  const int nb = p.nb;
  TcbRing ring;
  ring.base = acc_tile_base() + S::acc_bytes(nb);
  ring.stage_bytes = S::stage_bytes(nb, PASSES);
  ring.stages = p.stages;
  ring.bars = ring.base + (uint32_t)p.stages * ring.stage_bytes;
  const uint32_t acc_full = ring.bars + S::ACC_BARS_OFF;  // the families are stored: the epilogue may read
  const uint32_t acc_empty = acc_full + 8u;              // the epilogue is done: the MMA warps may store

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.num_m_tiles * p.num_n_tiles;
  const uint32_t tile_addr = acc_tile(2 * nb);
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(ring.full(s), 1);
      mbar_init(ring.empty(s), 8);  // one arrival per MMA warp
    }
    mbar_init(acc_full, TC_CONSUMER_THREADS);
    mbar_init(acc_empty, TC_CONSUMER_THREADS);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 8) {
    // ===================== MMA warps (thread 0: also the TMA loads) =====================
    // this CTA's K blocks, in order: block b is K block b % kb_n of its tile b / kb_n, in ring stage b % stages
    const int my_tiles = blockIdx.x < num_tiles ? (num_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const int total = my_tiles * p.kb_n;
    auto load = [&](int b) {
      const int tile = (int)blockIdx.x + (b / p.kb_n) * (int)gridDim.x;
      const int m_tile = tile / p.num_n_tiles;
      tcb_load_block<R, PASSES, 4>(&tm_a, &tm_b, ring, b % p.stages, m_tile, tile - m_tile * p.num_n_tiles,
                                   b % p.kb_n, nb);
    };
    // The tile loop keeps one counter, this CTA's tile index t: the tile, the refilled block and the acc_empty
    // parity derive from it (each counter beside the 88 accumulators is a register the K loop may have to spill)
    int t = 0;
    auto refill = [&](int kb) {  // K block kb of tile t has been released by this warp
      if (threadIdx.x == 0) {
        const int b = t * p.kb_n + kb;
        mbar_wait(ring.empty(b % p.stages), (uint32_t)(b / p.stages) & 1u);
        if (b + p.stages < total) load(b + p.stages);
      }
      __syncwarp();  // warp 0 reconverges before its next wgmma
    };
    if (threadIdx.x == 0) {
      prefetch_tmap(&tm_a);
      prefetch_tmap(&tm_b);
      for (int b = 0; b < p.stages && b < total; ++b) load(b);
    }
    float acc[TCB_WS_NB_MAX];
    int stage = 0;
    uint32_t phase = 0;
    for (; t < my_tiles; ++t) {
      const int n_tile = ((int)blockIdx.x + t * (int)gridDim.x) % p.num_n_tiles;
#pragma unroll
      for (int i = 0; i < TCB_WS_NB_MAX; ++i) acc[i] = 0.f;
      // the butterfly on the registers, then the families stored once the epilogue has read the previous tile
      // (the first wait passes)
      auto wait = [&] { mbar_wait(acc_empty, ((uint32_t)t & 1u) ^ 1u); };
      switch (nb) {  // nb = 32 .. TCB_WS_NB_MAX in steps of 8
#define NNAB_TCB_CASE(N) \
  case N:                                                                                                   \
    tcb_poly_tile<N, PASSES, 0>(p, acc, ring, n_tile, warp, lane, stage, phase, wait, refill); \
    break;
        NNAB_TCB_CASE(32) NNAB_TCB_CASE(40) NNAB_TCB_CASE(48) NNAB_TCB_CASE(56) NNAB_TCB_CASE(64)
        NNAB_TCB_CASE(72) NNAB_TCB_CASE(80) NNAB_TCB_CASE(88)
#undef NNAB_TCB_CASE
        default: break;
      }
      mbar_arrive(acc_full);
    }
    return;
  }

  // ===================== epilogue warps =====================
  const int ew = warp - 8;
  int4* acts = reinterpret_cast<int4*>(nnab_dyn_smem + (ring.bars + S::BAR_BYTES - smem_u32(nnab_dyn_smem))) +
               ew * TCB_WS_ACTS;
  uint32_t full_phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m_tile = tile / p.num_n_tiles;
    const int n_tile = tile - m_tile * p.num_n_tiles;
    if constexpr (FMT == 5) tcb_stage_actions(p, n_tile, ew & 3, ew >> 2, lane, acts);
    mbar_wait(acc_full, full_phase);
    full_phase ^= 1u;
    tcb_epilogue<FMT, R, 4, FMT == 5>(p, tile_addr, m_tile, n_tile, ew & 3, ew >> 2, lane,
                                      ring.bars + S::HANDOVER_OFF, acts);
    mbar_arrive(acc_empty);
  }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
template <int FMT, int R, int PASSES, int PH>
static int launch_tcb_fmt(const CUtensorMap& ma, const CUtensorMap& mb, const TcbParams& prm, int grid,
                          cudaStream_t stream) {
  using S = TcbSmem;
  // Four phases, fused filterbank (FMT 5) or operand planes (FMT 9), up to TCB_WS_NB_MAX packed bins per tile:
  // separate MMA and epilogue warps (wider tiles need more accumulator registers than the MMA warps have).  The plain STFT formats
  // keep framed_tcb_kernel: their epilogue is shorter than the MMA warps' share of a tile, and with separate roles
  // Magnitude STFT-2048 measured 7 % slower, where the Mel, MFCC and Gammatone workloads run 3-5 % faster.
  constexpr bool WS = PH == 4 && (FMT == 5 || FMT == 9);
  TcbParams q = prm;
  if (!WS || prm.nb > TCB_WS_NB_MAX) {
    q.stages = S::stages(prm.nb, PASSES);
    return launch_persistent<framed_tcb_kernel<FMT, R, PASSES, PH>>(grid, TC_KERNEL_THREADS, S::total(prm.nb, PASSES),
                                                                    S::LIMIT, stream, ma, mb, q);
  }
  if constexpr (WS) {
    const uint32_t extra = FMT == 5 ? TCB_WS_ACT_BYTES : 0;
    q.stages = S::stages(prm.nb, PASSES, extra);
    const int rc = launch_persistent<framed_tcb_ws_kernel<FMT, R, PASSES>>(grid, TCB_WS_THREADS,
                                                                           S::total(prm.nb, PASSES, extra), S::LIMIT,
                                                                           stream, ma, mb, q);
    if (rc == NNAB_OK) count_block_ws_launch();
    return rc;
  }
  return NNAB_EINVAL;  // (not reached)
}

template <int R, int PASSES, int PH>
static int launch_tcb(int fmt, const CUtensorMap& ma, const CUtensorMap& mb, const TcbParams& prm, int grid,
                      cudaStream_t stream) {
  switch (fmt) {
    case NNAB_FMT_MAGNITUDE: return launch_tcb_fmt<0, R, PASSES, PH>(ma, mb, prm, grid, stream);
    case NNAB_FMT_COMPLEX: return launch_tcb_fmt<1, R, PASSES, PH>(ma, mb, prm, grid, stream);
    case NNAB_FMT_PHASE_ANGLE: return launch_tcb_fmt<2, R, PASSES, PH>(ma, mb, prm, grid, stream);
    case FMT_POWER: return launch_tcb_fmt<4, R, PASSES, PH>(ma, mb, prm, grid, stream);
    case FMT_FBANK: return launch_tcb_fmt<5, R, PASSES, PH>(ma, mb, prm, grid, stream);
    case FMT_PLANES: return launch_tcb_fmt<9, R, PASSES, PH>(ma, mb, prm, grid, stream);
    default: return NNAB_EINVAL;
  }
}

template <int PH>
static int launch_tcb_ph(int R, int passes, int fmt, const CUtensorMap& ma, const CUtensorMap& mb,
                         const TcbParams& prm, int grid, cudaStream_t stream) {
  if (passes == 2)
    return R == 4 ? launch_tcb<4, 2, PH>(fmt, ma, mb, prm, grid, stream)
                  : launch_tcb<2, 2, PH>(fmt, ma, mb, prm, grid, stream);
  return R == 4 ? launch_tcb<4, 3, PH>(fmt, ma, mb, prm, grid, stream)
                : launch_tcb<2, 3, PH>(fmt, ma, mb, prm, grid, stream);
}

int launch_framed_tc_block(const FramedProblem& q, const void* packed, void* workspace,
                           size_t ws_bytes, cudaStream_t stream) {
  int n_fft = 0, hop = 0;
  if (packed_kind(packed, &n_fft, &hop) != PACK_BLOCK) return NNAB_EINVAL;
  // the basis was packed for exactly this transform: anything else is a caller bug
  if (n_fft != q.K || hop != q.hop || q.F != q.K / 2 + 1) return NNAB_EINVAL;
  if (q.presplit != nullptr || q.h_k_begin != nullptr || q.scale != nullptr || q.scale_all != 1.f)
    return NNAB_EINVAL;
  switch (q.fmt) {
    case NNAB_FMT_MAGNITUDE: case NNAB_FMT_COMPLEX: case NNAB_FMT_PHASE_ANGLE: case FMT_POWER:
      if (q.bin_offset != 0 || q.out_bins < q.F) return NNAB_EINVAL;
      break;
    case FMT_FBANK:
      if (q.fb_table == nullptr || q.n_fb <= 0) return NNAB_EINVAL;
      break;
    case FMT_PLANES:
      if (q.out == nullptr || q.planes_pitch <= 0 || q.planes_pitch % 8 != 0 || q.planes_stride <= 0 ||
          q.planes_stride % 8 != 0 || ((uintptr_t)q.out & 15u) != 0)
        return NNAB_EINVAL;
      break;
    default: return NNAB_EINVAL;
  }
  const size_t need = tc_workspace_bytes(q.B, q.L, q.K, q.hop, q.pad);
  if (workspace == nullptr || ws_bytes < need) return NNAB_EWORKSPACE;
  if (q.B > 65535) return NNAB_EUNSUPPORTED;

  const int R = q.K / q.hop;
  const bool poly = block_poly4(q.hop);
  const int PH = poly ? 4 : 1;
  const int Fb = block_basis_F(q.K, q.hop), Kb = block_basis_K(q.hop);  // the GEMM's packed bins and K
  const SplitGeom g = split_geom(q.B, q.L, q.K, q.hop, q.pad);
  __nv_bfloat16* planes =
      reinterpret_cast<__nv_bfloat16*>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  int rc = tc_problem_split(q, planes, stream, poly ? TC_SPLIT_POLY4 : TC_SPLIT_PLAIN);
  if (rc) return rc;
  // a bf16 waveform has an all-zero lo plane: the xlo * whi pass would add exact zeros
  const int passes = (q.x_dtype == NNAB_DTYPE_BF16) ? 2 : 3;

  int sms;
  if ((rc = usable_sms(&sms))) return rc;

  int nb = block_choose_nb(Fb);
  if (q.fmt == FMT_FBANK && q.fb_steps != nullptr && poly && q.fb_poly_tile != 0) {
    // run-to-run identical filterbank sums: the table builder replayed the four-phase range cuts (family
    // seams and tiles; the warp parts hand over inside the CTA) and chose the cheapest width that gives
    // every filter <= 2 partial sums
    nb = q.fb_poly_tile;
  } else if (q.fmt == FMT_FBANK && q.fb_steps != nullptr && !poly && q.fb_nb_mask != 0) {
    // run-to-run identical filterbank sums: with at most two partial sums per filter the atomic
    // adds commute.  The table builder replayed the range cuts for every tile width; take the
    // cheapest width that qualifies (fewest padded columns), else keep the default.
    int best = -1, best_cost = 1 << 30;
    for (int i = 0; i < 13; ++i) {
      if (!((q.fb_nb_mask >> i) & 1)) continue;
      const int c = 32 + 8 * i;
      const int cost = block_n_tiles(q.F, c) * (c + 6);
      if (cost < best_cost) { best_cost = cost; best = c; }
    }
    if (best > 0) nb = best;
  }
  if (nb < 32 || nb > 128 || nb % 8 != 0) return NNAB_EINVAL;
  const int c_split = (nb / 8) / TCB_PARTS;  // the two warp parts split the chunks evenly (>= 2: both own some)
  const int n_tiles = block_n_tiles(Fb, nb);
  const int p_rows = block_p_rows(Fb);
  CUtensorMap ma, mb;
  if (poly) {
    // A as (k < hop / 4, block row, phase, plane): 16-row boxes of two phases x 8 block rows (tcb_load_block).
    // The block-row dimension is the only one a box can leave, so the rows past the last block read as zeros.
    const uint64_t dims[4] = {(uint64_t)Kb, (uint64_t)g.rows, 4, 2};
    const uint64_t strides[3] = {(uint64_t)q.hop * 2, (uint64_t)Kb * 2, (uint64_t)g.plane_stride * 2};
    const uint32_t box[3] = {TCB_BK, 8, 2};
    rc = encode_4d(&ma, planes, dims, strides, box, TCB_BK);
    if (rc) return rc;
    // B: one box of 2 nb interleaved re / im rows per plane
    rc = encode_3d(&mb, const_cast<void*>(packed), (uint64_t)Kb, (uint64_t)(2 * p_rows), 2, (uint64_t)Kb * 2,
                   (uint64_t)(2 * p_rows) * Kb * 2, TCB_BK, (uint32_t)(2 * nb), TCB_BK);
  } else {
    rc = encode_3d(&ma, planes, (uint64_t)q.hop, (uint64_t)g.rows, 2, (uint64_t)q.hop * 2,
                   (uint64_t)g.plane_stride * 2, TCB_BK, 32, TCB_BK);
    if (rc) return rc;
    rc = encode_3d(&mb, const_cast<void*>(packed), (uint64_t)Kb, (uint64_t)p_rows, 4,
                   (uint64_t)Kb * 2, (uint64_t)p_rows * Kb * 2, TCB_BK, (uint32_t)nb, TCB_BK);
  }
  if (rc) return rc;

  TcbParams prm{};
  const int rows_per_tile = poly ? 33 - R : 4 * (33 - R);  // block rows (= frames) an M tile advances
  prm.num_m_tiles = (int)ceil_div64(g.nv, rows_per_tile);
  prm.num_n_tiles = n_tiles;
  prm.nb = nb;
  prm.kb_n = Kb / TCB_BK;
  prm.c_split = c_split;
  prm.fam_M = poly ? q.K / 4 : 0;
  prm.twiddle = poly ? reinterpret_cast<const float2*>((const char*)packed + block_twiddle_offset(q.K, q.hop))
                     : nullptr;
  prm.tw_rows = p_rows;
  prm.nv = g.nv;
  prm.t_slots = g.t_slots;
  prm.T = q.T;
  prm.epi = epilogue_of(q);
  if (q.fmt == FMT_PLANES && (int64_t)n_tiles * PH * nb > q.planes_pitch) return NNAB_EINVAL;
  const int64_t tiles = (int64_t)prm.num_m_tiles * n_tiles;
  const int grid = (int)(tiles < sms ? tiles : sms);
  add_exec_flops(passes * 2.0 * (double)tiles * TC_BM * (2 * nb) * Kb);
  rc = poly ? launch_tcb_ph<4>(R, passes, q.fmt, ma, mb, prm, grid, stream)
            : launch_tcb_ph<1>(R, passes, q.fmt, ma, mb, prm, grid, stream);
  if (rc == NNAB_OK && q.route != nullptr) *q.route = ROUTE_BLOCK;
  return rc;
}

}  // namespace nnab
