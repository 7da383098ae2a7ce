// wgmma / TMA framed contraction for sm_90a.
//
//   D[g, n] = sum_k A[g, k] * W[n, k]        g = virtual frame, n = basis row
//
// * A is never materialised: the padded waveform is written once as bf16 hi/lo
//   planes (pad_split_kernel) with a per-clip pitch that is a multiple of hop, so
//   the frames of the WHOLE batch form one Toeplitz matrix whose row g starts at
//   element g*hop.  TMA reads 128-frame x 64 tiles of it straight into
//   128B-swizzled shared memory (either as a plain (rows x hop) matrix when
//   64 | hop, or through an overlapping-stride tensor map otherwise).
// * W (basis) is pre-split into bf16 hi/lo planes, re rows and NEGATED im rows
//   grouped per N tile (pack_basis_kernel).
// * fp32 parity on bf16 tensor cores: x*w ~= xhi*whi + xlo*whi + xhi*wlo
//   (3 wgmma passes into one fp32 register accumulator; error ~2^-16).
// * Warp roles (288 threads, 1 CTA/SM, persistent over output tiles, tc_ptx.cuh):
//     warps 0-7  two wgmma warpgroups (64 tile rows each), then the epilogue from the shared-memory
//                accumulator tile -> magnitude/complex/phase/power -> coalesced stores in the
//                reference's (B, F, T[,2]) layout
//     warp 8     TMA producer (full/empty mbarrier ring)
#include <cuda.h>
#include <mutex>
#include <unordered_map>
#include <algorithm>
#include <vector>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdlib.h>
#include <type_traits>

#include "common.cuh"
#include "epilogue.cuh"
#include "tc_ptx.cuh"
#include "tc_host.cuh"
#include "tc_decim.cuh"

namespace nnab {

constexpr int TC_MAX_N_TILES = 128;


// N tile (columns = re + im rows of bn/2 bins): minimise padded columns among the widths that need at most
// TC_MAX_N_TILES tiles (256 when none does: tc_supported then refuses the basis).
static int choose_bn(int F) {
  const int cols = 2 * F;
  if (cols <= 256) return round_up_i(cols, 16) < 32 ? 32 : round_up_i(cols, 16);
  int best = 256, best_total = round_up_i(cols, 256);
  for (int bn = 240; bn >= 128; bn -= 16) {
    const int tiles = (cols + bn - 1) / bn;
    if (tiles > TC_MAX_N_TILES) break;  // narrower widths need more tiles still
    if (tiles * bn < best_total) { best_total = tiles * bn; best = bn; }
  }
  return best;
}

int tc_tile_n(int F) { return choose_bn(F > 0 ? F : 1); }

size_t tc_packed_bytes(int F, int K) {
  const int bn = choose_bn(F);
  const int n_tiles = (2 * F + bn - 1) / bn;
  const size_t rows = (size_t)n_tiles * bn;
  const size_t kpad = (size_t)round_up_i(K, 64);
  return 2 * rows * kpad * sizeof(__nv_bfloat16);
}

// ---------------------------------------------------------------------------
// geometry of the split / padded signal workspace
// ---------------------------------------------------------------------------

// Frames t = p, p + np, p + 2 np, ... (phase p of np = 8 / gcd(hop, 8)) start at
// multiples of hop * np, which is always a multiple of 8 samples = 16 bytes in
// bf16: every hop is served by TMA, one pass per phase over a signal shifted by
// p * hop samples.
static int gcd_i(int a, int b) { return b == 0 ? a : gcd_i(b, a % b); }
int num_phases(int hop) { return 8 / gcd_i(hop, 8); }

SplitGeom split_geom(int64_t B, int64_t L, int K, int hop, int pad) {
  const int hop_eff = hop * num_phases(hop);
  SplitGeom g;
  g.t_slots = (L + 2 * (int64_t)pad + hop_eff - 1) / hop_eff;
  g.nv = B * g.t_slots;
  const int kpad = round_up_i(K, 64);
  g.rows = g.nv + (kpad + hop_eff - 1) / hop_eff + 1;
  g.plane_stride = (g.rows * hop_eff + 63) / 64 * 64;
  return g;
}

size_t tc_workspace_bytes(int64_t B, int64_t L, int K, int hop, int pad) {
  const SplitGeom g = split_geom(B, L, K, hop, pad);
  return (size_t)(2 * g.plane_stride) * sizeof(__nv_bfloat16) + 256;
}

int tc_istft_bn(int n_fft) { return n_fft >= 256 ? 256 : (round_up_i(n_fft, 16) < 32 ? 32 : round_up_i(n_fft, 16)); }

// The FMT_OLA GEMM's N axis is the frame's F_out output samples in tc_istft_bn(F_out)-wide tiles, each with
// its own kb_begin / kb_end entry (so F_out <= TC_MAX_N_TILES x 256 = 32768).  Its callers pass no per-bin tap
// support, so every tile runs all round_up(K_gemm, 64) / 64 k-blocks.  Those are cut into chunks of at most 64
// k-blocks (4096 products per fp32 accumulator, as the dense kernel's split-K does), at most k_splits_hint of them;
// the overlap-add atomics sum the chunks.  A 24576-sample frame summed in one accumulator is 1e-4 off.
OlaPlan tc_ola_plan(int F_out, int K_gemm, int64_t M_rows, int k_splits_hint) {
  OlaPlan o{};
  if (F_out <= 0 || K_gemm <= 0 || M_rows < 0) return o;
  o.bn = tc_istft_bn(F_out);
  o.n_tiles = (F_out + o.bn - 1) / o.bn;
  o.supported = o.n_tiles <= TC_MAX_N_TILES;
  const int kpad = round_up_i(K_gemm, 64);
  const int nkb = kpad / 64;
  const int ks = (nkb + 63) / 64;  // <= nkb
  o.k_splits = ks < k_splits_hint ? ks : (k_splits_hint > 1 ? k_splits_hint : 1);
  o.exec_flops = 3.0 * 2.0 * (double)ceil_div64(M_rows, TC_BM) * TC_BM * ((double)o.n_tiles * o.bn) * kpad;
  return o;
}

bool tc_supported(const FramedProblem& p, const void* packed) {
  if (p.hop <= 0 || p.K < 16) return false;
  // (pre-split planes are laid out by the caller, which guarantees >= 1 valid frame)
  if (p.presplit == nullptr && p.L + 2 * (int64_t)p.pad < p.K) return false;
  const SplitGeom g = split_geom(p.B > 0 ? p.B : 1, p.L, p.K, p.hop, p.pad);
  if (g.rows >= (1ll << 31) || g.plane_stride >= (1ll << 38)) return false;
  if (p.fmt == FMT_OLA) return tc_ola_plan(p.F, p.K, g.nv, p.k_splits_hint).supported;
  // a block-partial basis runs on framed_tcb_kernel, whose nb-wide N tiles tc_block_shape_ok bounds (35 at
  // n_fft = 32768); the dense kernel's N-tile limit below would send n_fft = 24576 and 32768 to the SIMT kernel
  if (packed != nullptr && packed_kind(packed) == PACK_BLOCK) return tc_block_shape_ok(p.K, p.hop);
  const int bn = choose_bn(p.F);
  if ((2 * p.F + bn - 1) / bn > TC_MAX_N_TILES) return false;
  return true;
}

// ---------------------------------------------------------------------------
// pre-pass kernels
// ---------------------------------------------------------------------------

// Waveform samples as fp32: exact for all three sample types.  The planes are then a function of the fp32
// value only, so a 16-bit waveform gives the bytes its fp32 upcast gives (bf16: lo = 0; fp16: 11 significant
// bits, exactly hi + lo).
__device__ __forceinline__ float sample_f32(float v) { return v; }
__device__ __forceinline__ float sample_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float sample_f32(__half v) { return __half2float(v); }

// Samples i0 .. i0 + 7 of the centre-padded clip xb (L samples, `pad` on each side) as fp32.  Runs of 8 inside
// the clip whose address is 16-byte aligned are read with 16-byte loads.
template <typename Tx>
__device__ __forceinline__ void padded_samples8(const Tx* __restrict__ xb, int64_t L, int pad, int pad_mode,
                                                int64_t i0, float (&v)[8]) {
  const int64_t j0 = i0 - pad;
  if (j0 >= 0 && j0 + 8 <= L && (reinterpret_cast<uintptr_t>(xb + j0) & 15u) == 0) {
    constexpr int PER = 16 / (int)sizeof(Tx);  // samples per 16-byte load
#pragma unroll
    for (int c = 0; c < 8 / PER; ++c) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(xb + j0) + c);
      const Tx* s = reinterpret_cast<const Tx*>(&u);
#pragma unroll
      for (int e = 0; e < PER; ++e) v[c * PER + e] = sample_f32(s[e]);
    }
    return;
  }
  const int64_t padded_len = L + 2 * (int64_t)pad;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int64_t i = i0 + e;
    v[e] = 0.f;
    if (i < padded_len) {
      int64_t j = i - pad;
      if (j < 0) j = (pad_mode == NNAB_PAD_REFLECT) ? -j : -1;
      else if (j >= L) j = (pad_mode == NNAB_PAD_REFLECT) ? 2 * (L - 1) - j : -1;
      if (j >= 0 && j < L) v[e] = sample_f32(__ldg(xb + j));
    }
  }
}

// Slot position -> sample of the clip slot.  poly_hop = 0: the identity.  poly_hop = hop (a multiple of 128):
// every hop-sized block is stored in polyphase order, position q * hop / 4 + m holding sample 4 m + q
// (TC_SPLIT_POLY4, the block-partial kernel's four-phase layout).  8 consecutive positions stay in one phase.
__device__ __forceinline__ int64_t split_src(int64_t i, int poly_hop) {
  if (poly_hop == 0) return i;
  const int64_t g = i / poly_hop;
  const int r = (int)(i - g * poly_hop), kq = poly_hop >> 2;
  const int q = r / kq;
  return g * poly_hop + 4 * (r - q * kq) + q;
}

// One thread = 8 consecutive positions of one clip's slot region (16-byte stores).
template <typename Tx>
__global__ void __launch_bounds__(256) pad_split_kernel(
    const Tx* __restrict__ x, int64_t L, int64_t x_pitch, int pad, int pad_mode, int shift,
    int64_t clip_pitch, int64_t plane_stride, int poly_hop, __nv_bfloat16* __restrict__ planes) {
  const int64_t b = blockIdx.y;
  const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i0 >= clip_pitch) return;
  float v[8];
  if (poly_hop == 0) {
    padded_samples8(x + b * x_pitch, L, pad, pad_mode, i0 + shift, v);  // i0 + shift: index into the padded clip
  } else {
    // samples 4 m + q .. 4 (m + 7) + q of one block: a stride-4 gather (the warp's other phases hit in L1)
    const Tx* __restrict__ xb = x + b * x_pitch;
    const int64_t s0 = split_src(i0, poly_hop) + shift;
    const int64_t padded_len = L + 2 * (int64_t)pad;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int64_t i = s0 + 4 * e;
      v[e] = 0.f;
      if (i < padded_len) {
        int64_t j = i - pad;
        if (j < 0) j = (pad_mode == NNAB_PAD_REFLECT) ? -j : -1;
        else if (j >= L) j = (pad_mode == NNAB_PAD_REFLECT) ? 2 * (L - 1) - j : -1;
        if (j >= 0 && j < L) v[e] = sample_f32(__ldg(xb + j));
      }
    }
  }
  __align__(16) __nv_bfloat16 hi[8];
  __align__(16) __nv_bfloat16 lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) split_bf16(v[e], hi[e], lo[e]);
  const int64_t o = b * clip_pitch + i0;
  *reinterpret_cast<uint4*>(planes + o) = *reinterpret_cast<const uint4*>(hi);
  *reinterpret_cast<uint4*>(planes + plane_stride + o) = *reinterpret_cast<const uint4*>(lo);
}

// pad_split_kernel on a push's virtual clips (ChunkSource): row b builds the clip of lane b, each sample taken
// from its fp32 carry ring row or its chunk row, with the reflect / constant centre padding of its whole stream
// at the two ends.  The planes of frame t0 + j are then those the whole-clip pre-pass writes for the lane's frame
// frames + t0 + j; the row's samples past what its own frames read are zeros.  A row with frames never mirrors
// past its samples on the left, nor further than pad on the right; a device pool's row without frames may, and
// reads nothing there.
template <typename Tx>
__global__ void __launch_bounds__(256) chunk_split_kernel(
    ChunkSource c, const Tx* __restrict__ chunk, int shift, int64_t clip_pitch, int64_t plane_stride,
    int poly_hop, __nv_bfloat16* __restrict__ planes) {
  const int64_t b = blockIdx.y;
  const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i0 >= clip_pitch) return;
  nnab_stream_lane ln = c.shared;
  ln.slot = b;
  if (c.lanes != nullptr) ln = c.lanes[b];
  const int64_t received = ln.received, total = ln.received + ln.n, origin = ln.frames * c.hop - c.pad;
  const float* __restrict__ ring = c.ring + ln.slot * c.ring_pitch;
  const Tx* __restrict__ xb = chunk + ln.slot * c.chunk_pitch;
  const bool reflect = c.pad_mode == NNAB_PAD_REFLECT;
  const int64_t s0 = split_src(i0, poly_hop) + shift;
  const int step = poly_hop ? 4 : 1;  // the 8 positions of a thread: consecutive samples, or one phase
  __align__(16) __nv_bfloat16 hi[8];
  __align__(16) __nv_bfloat16 lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int64_t i = s0 + step * e;
    float v = 0.f;
    if (i < c.length) {
      int64_t r = origin + i;
      bool live = true;
      if (r < 0) {
        if (reflect) r = -r; else live = false;
        if (r >= total) live = false;
      } else if (r >= total) {
        // the clip runs past the row's own right padding (the longest row sets the length): zeros there
        if (ln.end && reflect && r - total < c.pad) r = 2 * (total - 1) - r; else live = false;
      }
      if (live) v = r < received ? __ldg(ring + r % c.ring_len) : sample_f32(__ldg(xb + (r - received)));
    }
    split_bf16(v, hi[e], lo[e]);
  }
  const int64_t o = b * clip_pitch + i0;
  *reinterpret_cast<uint4*>(planes + o) = *reinterpret_cast<const uint4*>(hi);
  *reinterpret_cast<uint4*>(planes + plane_stride + o) = *reinterpret_cast<const uint4*>(lo);
}

// Raw samples [from, received + n) of lane b's chunk row into its carry ring row, from = chunk_carry_start after
// the lane's frames and never before its first new sample (the host's rule, stream_step).  Runs after every
// kernel of the push that reads the ring (same stream), and never overwrites a sample the next push reads: the
// ring holds ring_len >= the longest carry.
template <typename Tx>
__global__ void __launch_bounds__(256) chunk_carry_kernel(ChunkSource c, const Tx* __restrict__ chunk) {
  nnab_stream_lane ln = c.shared;
  ln.slot = blockIdx.y;
  if (c.lanes != nullptr) ln = c.lanes[blockIdx.y];
  const int64_t total = ln.received + ln.n;
  const int64_t keep = chunk_carry_start(total, lane_frames_after(ln, c.K, c.hop, c.pad, c.pad_mode), c.hop, c.pad);
  const int64_t from = keep > ln.received ? keep : ln.received;
  const int64_t r = from + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= total) return;
  const_cast<float*>(c.ring)[ln.slot * c.ring_pitch + r % c.ring_len] =
      sample_f32(__ldg(chunk + ln.slot * c.chunk_pitch + (r - ln.received)));
}

// Stream pools: frames t >= count of row i of out (A, rows, T, cols) are exact zeros (the row's clip is the
// batch's longest, so the transform also computed frames its stream has not completed).
__global__ void __launch_bounds__(256) pool_mask_kernel(ChunkSource c, float* __restrict__ out, int64_t rows,
                                                        int64_t T, int cols) {
  const nnab_stream_lane ln = c.lanes[blockIdx.y];
  const int64_t count = lane_frames_after(ln, c.K, c.hop, c.pad, c.pad_mode) - ln.frames;
  if (count >= T) return;
  const int64_t row_len = (T - count) * cols;  // the tail of each of the `rows` rows
  float* __restrict__ o = out + (int64_t)blockIdx.y * rows * T * cols;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < rows * row_len;
       k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = k / row_len;
    o[r * T * cols + count * cols + (k - r * row_len)] = 0.f;
  }
}

// ---- device pools (DESIGN §3.10 "Device pools"): one thread per slot --------------------------------------
__global__ void __launch_bounds__(128) device_pool_plan_kernel(
    int64_t slots, int64_t* __restrict__ counters, const int32_t* __restrict__ lengths,
    const uint8_t* __restrict__ end, int32_t* __restrict__ errors, int64_t* __restrict__ info,
    int32_t* __restrict__ counts, nnab_stream_lane* __restrict__ lanes, int64_t chunk, int K, int hop, int pad,
    int pad_mode) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= slots) return;
  device_pool_slot(s, slots, counters, lengths, end, errors, info, counts, lanes, chunk, K, hop, pad, pad_mode);
}

__global__ void __launch_bounds__(128) device_istft_plan_kernel(
    int64_t slots, int64_t* __restrict__ counters, const int32_t* __restrict__ frame_counts,
    const uint8_t* __restrict__ end, const int64_t* __restrict__ length, int32_t* __restrict__ errors,
    int64_t* __restrict__ info, int32_t* __restrict__ counts, nnab_istft_lane* __restrict__ lanes, int64_t t,
    int n_fft, int hop, int center) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= slots) return;
  device_istft_slot(s, slots, counters, frame_counts, end, length, errors, info, counts, lanes, t, n_fft, hop,
                    center);
}

__global__ void __launch_bounds__(128) device_pool_reset_kernel(int64_t slots, int64_t* __restrict__ counters,
                                                                int32_t* __restrict__ errors,
                                                                int64_t* __restrict__ info,
                                                                const uint8_t* __restrict__ mask) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= slots || (mask != nullptr && mask[s] == 0)) return;
  counters[s] = counters[slots + s] = counters[2 * slots + s] = 0;
  errors[s] = NNAB_LANE_OK;
  info[2 * s] = info[2 * s + 1] = 0;
}

int tc_device_pool_plan(int64_t slots, int64_t* counters, const int32_t* lengths, const uint8_t* end,
                        int32_t* errors, int64_t* info, int32_t* counts, nnab_stream_lane* lanes, int64_t chunk,
                        int K, int hop, int pad, int pad_mode, cudaStream_t stream) {
  device_pool_plan_kernel<<<(unsigned)ceil_div64(slots, 128), 128, 0, stream>>>(
      slots, counters, lengths, end, errors, info, counts, lanes, chunk, K, hop, pad, pad_mode);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

int tc_device_istft_plan(int64_t slots, int64_t* counters, const int32_t* frame_counts, const uint8_t* end,
                         const int64_t* length, int32_t* errors, int64_t* info, int32_t* counts,
                         nnab_istft_lane* lanes, int64_t t, int n_fft, int hop, int center, cudaStream_t stream) {
  device_istft_plan_kernel<<<(unsigned)ceil_div64(slots, 128), 128, 0, stream>>>(
      slots, counters, frame_counts, end, length, errors, info, counts, lanes, t, n_fft, hop, center);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

int tc_device_pool_reset(int64_t slots, int64_t* counters, int32_t* errors, int64_t* info, const uint8_t* mask,
                         cudaStream_t stream) {
  device_pool_reset_kernel<<<(unsigned)ceil_div64(slots, 128), 128, 0, stream>>>(slots, counters, errors, info,
                                                                                   mask);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

// ---- pyramid pools (DESIGN §3.10 "Pyramid pools"): the kernels that know where each row's samples come from --
// The (signal, lane) descriptor table of a push: one thread per entry, pyr_lane_signal of the lane's counters.
// Without a lane table (a lock-step push) lane i is `shared` in slot i.
__global__ void __launch_bounds__(128) pyr_pool_plan_kernel(const PyrStream p,
                                                            const nnab_stream_lane* __restrict__ lanes,
                                                            const nnab_stream_lane shared, int64_t n_lanes,
                                                            int pad_mode, PyrLaneSig* __restrict__ table) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_lanes * p.n_sig) return;
  const int s = (int)(k / n_lanes);
  const int64_t i = k - s * n_lanes;
  if (lanes != nullptr) {  // two calls: one call on a selected lane copy spills a register
    table[k] = pyr_lane_signal(p, lanes[i], i, s, pad_mode);
    return;
  }
  nnab_stream_lane ln = shared;
  ln.slot = i;
  table[k] = pyr_lane_signal(p, ln, i, s, pad_mode);
}

// A device pyramid pool's plan launch: one thread per slot.
__global__ void __launch_bounds__(128) device_pyramid_plan_kernel(
    const PyrStream p, int64_t slots, int64_t* __restrict__ counters, const int32_t* __restrict__ lengths,
    const uint8_t* __restrict__ end, int32_t* __restrict__ errors, int64_t* __restrict__ info,
    int32_t* __restrict__ counts, nnab_stream_lane* __restrict__ lanes, int64_t chunk, int pad_mode) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= slots) return;
  device_pyramid_slot(s, slots, counters, lengths, end, errors, info, counts, lanes, chunk, p, pad_mode);
}

// chunk_split_kernel in the per-row descriptor mode (ChunkSource::rows): row b builds its own clip -- a FIR
// stage source from the lane's first 128-output row, or an octave clip from its first unreturned frame -- from its
// slot's ring row and its own source row, with its own counts, padding and end; past its samples, zeros.
template <typename Tx>
__global__ void __launch_bounds__(256) chunk_split_rows_kernel(
    ChunkSource c, const Tx* __restrict__ chunk, int shift, int64_t clip_pitch, int64_t plane_stride,
    int poly_hop, __nv_bfloat16* __restrict__ planes) {
  const int64_t b = blockIdx.y;
  const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i0 >= clip_pitch) return;
  const PyrLaneSig& d = c.rows[b];
  const int64_t origin = c.rows_oct ? d.oct_origin : d.fir_origin;
  const bool reflect = c.rows_oct && d.mode == NNAB_PAD_REFLECT;
  const bool at_end = !c.rows_oct || d.end;
  const float* __restrict__ ring = c.ring + d.slot * c.ring_pitch;
  const Tx* __restrict__ xb = chunk + d.src_row * c.chunk_pitch + d.base;
  const int64_t s0 = split_src(i0, poly_hop) + shift;
  const int step = poly_hop ? 4 : 1;
  __align__(16) __nv_bfloat16 hi[8];
  __align__(16) __nv_bfloat16 lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int64_t i = s0 + step * e;
    float v = 0.f;
    if (i < c.length) {
      int64_t r = origin + i;
      bool live = true;
      if (r < 0) {
        if (reflect) r = -r; else live = false;
        // a row without frames yet (or the zero lane of an idle device-pool slot) may mirror past its own
        // samples: those frames are masked, and nothing past R1 is there to read
        if (r >= d.R1) live = false;
      } else if (r >= d.R1) {
        if (at_end && reflect && r - d.R1 < c.pad) r = 2 * (d.R1 - 1) - r; else live = false;
      }
      if (live) v = r < d.R0 ? __ldg(ring + r % c.ring_len) : sample_f32(__ldg(xb + (r - d.R0)));
    }
    split_bf16(v, hi[e], lo[e]);
  }
  const int64_t o = b * clip_pitch + i0;
  *reinterpret_cast<uint4*>(planes + o) = *reinterpret_cast<const uint4*>(hi);
  *reinterpret_cast<uint4*>(planes + plane_stride + o) = *reinterpret_cast<const uint4*>(lo);
}

// chunk_carry_kernel in the descriptor mode: row b keeps [keep, R1) of its signal in its slot's ring row.
template <typename Tx>
__global__ void __launch_bounds__(256) chunk_carry_rows_kernel(ChunkSource c, const Tx* __restrict__ chunk) {
  const PyrLaneSig& d = c.rows[blockIdx.y];
  const int64_t r = d.keep + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= d.R1) return;
  const_cast<float*>(c.ring)[d.slot * c.ring_pitch + r % c.ring_len] =
      sample_f32(__ldg(chunk + d.src_row * c.chunk_pitch + d.base + (r - d.R0)));
}

// pool_mask_kernel with the count of each row from its descriptor.
__global__ void __launch_bounds__(256) rows_mask_kernel(const PyrLaneSig* __restrict__ desc,
                                                        float* __restrict__ out, int64_t rows, int64_t T, int cols) {
  const int64_t count = desc[blockIdx.y].count;
  if (count >= T) return;
  const int64_t row_len = (T - count) * cols;
  float* __restrict__ o = out + (int64_t)blockIdx.y * rows * T * cols;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < rows * row_len;
       k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = k / row_len;
    o[r * T * cols + count * cols + (k - r * row_len)] = 0.f;
  }
}

// The one sample-type dispatch (NNAB_DTYPE_*): f(samples) launches one kernel on x as fp32, bf16 or fp16
// samples, and the launch is checked.  (The deduced return type instantiates each call's kernels where the call
// stands, which keeps the module's kernel order.)
template <typename F>
static auto with_sample_type(int x_dtype, const void* x, F&& f) {
  if (x_dtype == NNAB_DTYPE_F32) f(static_cast<const float*>(x));
  else if (x_dtype == NNAB_DTYPE_BF16) f(static_cast<const __nv_bfloat16*>(x));
  else if (x_dtype == NNAB_DTYPE_F16) f(static_cast<const __half*>(x));
  else return NNAB_EINVAL;
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

static int launch_chunk_split(const ChunkSource& cs, int x_dtype, dim3 grid, int shift, int64_t clip_pitch,
                              int64_t plane_stride, int poly_hop, __nv_bfloat16* planes, cudaStream_t stream);

// The pre-pass of every tensor-core launcher: the planes of q's signal, shifted by `shift` samples.
static int launch_problem_split(const FramedProblem& q, dim3 grid, int shift, int64_t clip_pitch,
                                int64_t plane_stride, int poly_hop, __nv_bfloat16* planes, cudaStream_t stream) {
  if (q.chunk == nullptr)
    return with_sample_type(q.x_dtype, q.x, [&](auto* xs) {
      pad_split_kernel<<<grid, 256, 0, stream>>>(xs, q.L, q.x_pitch, q.pad, q.pad_mode, shift, clip_pitch,
                                                 plane_stride, poly_hop, planes);
    });
  return launch_chunk_split(*q.chunk, q.x_dtype, grid, shift, clip_pitch, plane_stride, poly_hop, planes, stream);
}

// Two differently padded split copies of the same batch in one pass over x (level 0 of
// the CQT pyramid: reflect-padded copy for the octave CQT + zero-margin copy for the FIR).
template <typename Tx>
__global__ void __launch_bounds__(256) pad_split2_kernel(
    const Tx* __restrict__ x, int64_t L, int64_t x_pitch,
    int pad_a, int mode_a, int64_t pitch_a, int64_t plane_a, __nv_bfloat16* __restrict__ pa,
    int pad_b, int mode_b, int64_t pitch_b, int64_t plane_b, __nv_bfloat16* __restrict__ pb) {
  const int64_t b = blockIdx.y;
  const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  const Tx* __restrict__ xb = x + b * x_pitch;
#pragma unroll
  for (int which = 0; which < 2; ++which) {
    const int pad = which ? pad_b : pad_a;
    const int mode = which ? mode_b : mode_a;
    const int64_t pitch = which ? pitch_b : pitch_a;
    const int64_t plane = which ? plane_b : plane_a;
    __nv_bfloat16* __restrict__ dst = which ? pb : pa;
    if (i0 >= pitch) continue;
    float v[8];
    padded_samples8(xb, L, pad, mode, i0, v);
    __align__(16) __nv_bfloat16 hi[8];
    __align__(16) __nv_bfloat16 lo[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) split_bf16(v[e], hi[e], lo[e]);
    const int64_t o = b * pitch + i0;
    *reinterpret_cast<uint4*>(dst + o) = *reinterpret_cast<const uint4*>(hi);
    *reinterpret_cast<uint4*>(dst + plane + o) = *reinterpret_cast<const uint4*>(lo);
  }
}

// packed[plane][tile*bn + part*bn/2 + j][k]; part 1 rows are NEGATED im rows.
__global__ void __launch_bounds__(256) pack_basis_kernel(
    const float* __restrict__ w_re, const float* __restrict__ w_im, int F, int K, int bn,
    int rows, int kpad, __nv_bfloat16* __restrict__ packed) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int k8 = kpad / 8;
  if (idx >= (int64_t)rows * k8) return;
  const int r = (int)(idx / k8);
  const int k0 = (int)(idx % k8) * 8;
  const int half = bn / 2;
  const int tile = r / bn, within = r % bn;
  const int part = within / half, j = within % half;
  const int f = tile * half + j;
  __align__(16) __nv_bfloat16 hi[8];
  __align__(16) __nv_bfloat16 lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = k0 + e;
    float v = 0.f;
    if (f < F && k < K)
      v = part == 0 ? __ldg(w_re + (int64_t)f * K + k) : -__ldg(w_im + (int64_t)f * K + k);
    split_bf16(v, hi[e], lo[e]);
  }
  const int64_t o = (int64_t)r * kpad + k0;
  *reinterpret_cast<uint4*>(packed + o) = *reinterpret_cast<const uint4*>(hi);
  *reinterpret_cast<uint4*>(packed + (int64_t)rows * kpad + o) = *reinterpret_cast<const uint4*>(lo);
}

static void tc_forget_packed(const void* packed) { mark_packed(packed, PACK_DENSE); }
bool tc_varn_basis_ok(int F, int K);
int tc_pack_basis_varn(const float* w_re, const float* w_im, int F, int K, void* packed,
                       cudaStream_t stream);

// layout: 0 = dense (always valid); 3 = 8-bin-group layout for the per-K-block-width / tall-A kernels
// (any basis with F <= 128; dense otherwise).
int tc_pack_basis_layout(const float* w_re, const float* w_im, int F, int K, int layout, void* packed,
                         cudaStream_t stream) {
  if (layout == 3 && tc_varn_basis_ok(F, K)) return tc_pack_basis_varn(w_re, w_im, F, K, packed, stream);
  if (layout != 0 && layout != 3) return NNAB_EINVAL;
  return tc_pack_basis(w_re, w_im, F, K, packed, stream);
}

int tc_pack_basis(const float* w_re, const float* w_im, int F, int K, void* packed,
                  cudaStream_t stream) {
  tc_forget_packed(packed);
  const int bn = choose_bn(F);
  const int n_tiles = (2 * F + bn - 1) / bn;
  const int rows = n_tiles * bn;
  const int kpad = round_up_i(K, 64);
  const int64_t threads = (int64_t)rows * (kpad / 8);
  pack_basis_kernel<<<(unsigned)ceil_div64(threads, 256), 256, 0, stream>>>(
      w_re, w_im, F, K, bn, rows, kpad, (__nv_bfloat16*)packed);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

// Decimating FIR as a framed contraction: frame t of the zero-padded level signal
// (sample m at plane offset 128 + m, hop 128*dec) against the banded Toeplitz rows
//   H[j][k] = fir[k - 1 - dec*j]        j = 0..127 outputs per frame
// gives y[128 t + j] = sum_m fir[m] x[dec*(128 t + j) + m - 127]
// (utils.py:73-100: conv1d(stride=dec, padding=127)).  Rows 0..63 sit in the "re" half
// of the single N tile and rows 64..127 in the "im" half (not negated).
int tc_fir_k(int taps, int dec) { return round_up_i(dec * 127 + taps + 1, 64); }
size_t tc_packed_fir_bytes(int taps, int dec) {
  return (size_t)2 * 128 * tc_fir_k(taps, dec) * sizeof(__nv_bfloat16);
}

__global__ void __launch_bounds__(256) pack_fir_kernel(const float* __restrict__ fir, int taps,
                                                       int dec, int kpad,
                                                       __nv_bfloat16* __restrict__ packed) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= 128 * kpad) return;
  const int r = idx / kpad, k = idx % kpad;
  const int m = k - 1 - dec * r;
  const float v = (m >= 0 && m < taps) ? __ldg(fir + m) : 0.f;
  __nv_bfloat16 hi, lo;
  split_bf16(v, hi, lo);
  packed[idx] = hi;
  packed[(int64_t)128 * kpad + idx] = lo;
}

int tc_pack_fir(const float* fir, int taps, int dec, void* packed, cudaStream_t stream) {
  tc_forget_packed(packed);  // dense rows: drop any stale layout entry of a recycled address
  const int kpad = tc_fir_k(taps, dec);
  pack_fir_kernel<<<(128 * kpad + 255) / 256, 256, 0, stream>>>(fir, taps, dec, kpad,
                                                               (__nv_bfloat16*)packed);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

void tc_split_geometry(int64_t B, int64_t L, int K, int hop, int pad, int64_t* t_slots,
                       int64_t* plane_stride, int* hop_eff) {
  const SplitGeom g = split_geom(B, L, K, hop, pad);
  if (t_slots) *t_slots = g.t_slots;
  if (plane_stride) *plane_stride = g.plane_stride;
  if (hop_eff) *hop_eff = hop * num_phases(hop);
}

// Zero [used, plane_stride) of both planes: the K-overhang rows past the last clip slot, which TMA reads and the
// basis multiplies by its zero padding (they must hold finite values).
static int zero_tail(__nv_bfloat16* planes, int64_t used, int64_t plane_stride, cudaStream_t stream) {
  const int64_t tail = plane_stride - used;
  for (int pl = 0; pl < 2 && tail > 0; ++pl)
    NNAB_CUDA_TRY(cudaMemsetAsync(planes + pl * plane_stride + used, 0, (size_t)tail * sizeof(__nv_bfloat16),
                                  stream));
  return NNAB_OK;
}

// phase-0 pad + split of a batch into caller-managed planes, in the given layout (TC_SPLIT_*)
int tc_problem_split(const FramedProblem& q, void* planes_v, cudaStream_t stream, int layout) {
  if (q.B > 65535) return NNAB_EUNSUPPORTED;
  if (layout != TC_SPLIT_PLAIN && (layout != TC_SPLIT_POLY4 || q.hop % 128 != 0)) return NNAB_EINVAL;
  const SplitGeom g = split_geom(q.B, q.L, q.K, q.hop, q.pad);
  const int hop_eff = q.hop * num_phases(q.hop);
  __nv_bfloat16* planes = (__nv_bfloat16*)planes_v;
  const int64_t clip_pitch = g.t_slots * hop_eff;
  int rc = zero_tail(planes, q.B * clip_pitch, g.plane_stride, stream);
  if (rc) return rc;
  dim3 grid((unsigned)ceil_div64(clip_pitch, 256 * 8), (unsigned)q.B);
  return launch_problem_split(q, grid, 0, clip_pitch, g.plane_stride, layout == TC_SPLIT_POLY4 ? q.hop : 0,
                              planes, stream);
}

int tc_pad_split(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch, int K, int hop, int pad,
                 int pad_mode, void* planes_v, cudaStream_t stream) {
  FramedProblem q{};
  q.x = x; q.x_dtype = x_dtype; q.B = B; q.L = L; q.x_pitch = x_pitch;
  q.K = K; q.hop = hop; q.pad = pad; q.pad_mode = pad_mode;
  return tc_problem_split(q, planes_v, stream, TC_SPLIT_PLAIN);
}

// pad + split into caller-defined geometry (clip pitch / plane stride in elements).  pad_split_kernel
// writes the whole [0, clip_pitch) slot of every clip (zeros past the padded signal); the tail
// [B * clip_pitch, plane_stride) is zeroed here.
int tc_pad_split_ex(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch, int pad, int pad_mode,
                    int64_t clip_pitch, int64_t plane_stride, void* planes_v, cudaStream_t stream) {
  if (B > 65535) return NNAB_EUNSUPPORTED;
  if (clip_pitch % 8 != 0 || plane_stride < B * clip_pitch) return NNAB_EINVAL;
  __nv_bfloat16* planes = (__nv_bfloat16*)planes_v;
  const int rc = zero_tail(planes, B * clip_pitch, plane_stride, stream);
  if (rc) return rc;
  dim3 grid((unsigned)ceil_div64(clip_pitch, 256 * 8), (unsigned)B);
  return with_sample_type(x_dtype, x, [&](auto* xs) {
    pad_split_kernel<<<grid, 256, 0, stream>>>(xs, L, x_pitch, pad, pad_mode, 0, clip_pitch, plane_stride, 0,
                                               planes);
  });
}

int tc_pad_split2(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch,
                  int K_a, int hop_a, int pad_a, int mode_a, void* planes_a,
                  int K_b, int hop_b, int pad_b, int mode_b, void* planes_b, cudaStream_t stream) {
  if (B > 65535) return NNAB_EUNSUPPORTED;
  const SplitGeom ga = split_geom(B, L, K_a, hop_a, pad_a);
  const SplitGeom gb = split_geom(B, L, K_b, hop_b, pad_b);
  const int64_t pitch_a = ga.t_slots * hop_a * num_phases(hop_a), pitch_b = gb.t_slots * hop_b * num_phases(hop_b);
  const int64_t pmax = pitch_a > pitch_b ? pitch_a : pitch_b;
  dim3 grid((unsigned)ceil_div64(pmax, 256 * 8), (unsigned)B);
  // the kernel writes the clip slots, [0, B * pitch) of each plane set; the tails past them are zeroed after
  int rc = with_sample_type(x_dtype, x, [&](auto* xs) {
    pad_split2_kernel<<<grid, 256, 0, stream>>>(xs, L, x_pitch, pad_a, mode_a, pitch_a, ga.plane_stride,
                                                (__nv_bfloat16*)planes_a, pad_b, mode_b, pitch_b,
                                                gb.plane_stride, (__nv_bfloat16*)planes_b);
  });
  if (rc) return rc;
  if ((rc = zero_tail((__nv_bfloat16*)planes_a, B * pitch_a, ga.plane_stride, stream))) return rc;
  return zero_tail((__nv_bfloat16*)planes_b, B * pitch_b, gb.plane_stride, stream);
}

// Zero every element of each clip's slot region outside [keep_lo, keep_hi) (both planes)
// plus the K-overhang tail: the parts of a level buffer the FIR epilogue never writes.
__global__ void __launch_bounds__(256) zero_margins_kernel(__nv_bfloat16* __restrict__ planes,
                                                           int64_t plane_stride, int64_t pitch,
                                                           int64_t keep_lo, int64_t keep_hi) {
  const int64_t b = blockIdx.y;
  const int64_t lo_n = keep_lo, hi_n = pitch - keep_hi;
  const int64_t n = lo_n + hi_n;
  const __nv_bfloat16 z = __float2bfloat16_rn(0.f);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pos = i < lo_n ? i : keep_hi + (i - lo_n);
    planes[b * pitch + pos] = z;
    planes[plane_stride + b * pitch + pos] = z;
  }
}

// zero [keep_hi, clip_pitch) and [0, keep_lo) of every clip slot (both planes) + the tail of the planes
int tc_zero_slots(void* planes_v, int64_t B, int64_t clip_pitch, int64_t plane_stride, int64_t keep_lo,
                  int64_t keep_hi, cudaStream_t stream) {
  if (B > 65535) return NNAB_EUNSUPPORTED;
  __nv_bfloat16* planes = (__nv_bfloat16*)planes_v;
  const int rc = zero_tail(planes, B * clip_pitch, plane_stride, stream);
  if (rc) return rc;
  if (keep_hi > clip_pitch) keep_hi = clip_pitch;
  if (keep_lo < 0) keep_lo = 0;
  const int64_t n = keep_lo + (clip_pitch - keep_hi);
  if (n <= 0) return NNAB_OK;
  int gx = (int)ceil_div64(n, 256);
  if (gx > 64) gx = 64;
  zero_margins_kernel<<<dim3(gx, (unsigned)B), 256, 0, stream>>>(planes, plane_stride, clip_pitch,
                                                                keep_lo, keep_hi);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

// ---------------------------------------------------------------------------
// inverse STFT (stft.py:15-63) as a plain GEMM on the framed kernel:
//   frame[g, n] = sum_k A[g, k] * Winv[n, k],  g = b*T + t,  k = (re | im) x frequency
// "hop = Kpad" rows: every frame is its own row, so the Toeplitz machinery degenerates to a
// row-major matrix.  The FMT_OLA epilogue windows the frame and overlap-adds it.
// ---------------------------------------------------------------------------
int tc_istft_k(int f_in) { return round_up_i(2 * f_in, 64); }
size_t tc_packed_istft_bytes(int n_fft, int f_in) {
  const int bn = tc_istft_bn(n_fft);
  const size_t rows = (size_t)((n_fft + bn - 1) / bn) * bn;
  return 2 * rows * tc_istft_k(f_in) * sizeof(__nv_bfloat16);
}

// Winv[n][f]        = KC[n][f] (+ KC[n][N-f] for a mirrored one-sided bin)          re part
// Winv[n][F_in + f] = -(KS[n][f] (- KS[n][N-f]))                                    im part
// i.e. the reference's extend_fbins (utils.py:63-70) folded into the kernels.
// With `transposed` the inputs are the FORWARD bases (f_in, n_fft) = wcos / wsin and the rows
// become W^T (the adjoint used by the input gradient): Winv[n][f] = wcos[f][n], -wsin[f][n].
__global__ void __launch_bounds__(256) pack_istft_kernel(const float* __restrict__ kc,
                                                         const float* __restrict__ ks, int n_fft,
                                                         int f_in, int onesided, int transposed,
                                                         int rows, int kpad,
                                                         __nv_bfloat16* __restrict__ packed) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)rows * kpad) return;
  const int n = (int)(idx / kpad), k = (int)(idx % kpad);
  float v = 0.f;
  if (n < n_fft && k < 2 * f_in) {
    const int part = k / f_in, f = k % f_in;
    const bool mirror = onesided && !transposed && f > 0 && f < n_fft - f && (n_fft - f) < n_fft;
    if (transposed) {
      v = part == 0 ? __ldg(kc + (int64_t)f * n_fft + n) : -__ldg(ks + (int64_t)f * n_fft + n);
    } else if (part == 0) {
      v = __ldg(kc + (int64_t)n * n_fft + f);
      if (mirror) v += __ldg(kc + (int64_t)n * n_fft + (n_fft - f));
    } else {
      v = __ldg(ks + (int64_t)n * n_fft + f);
      if (mirror) v -= __ldg(ks + (int64_t)n * n_fft + (n_fft - f));
      v = -v;
    }
  }
  __nv_bfloat16 hi, lo;
  split_bf16(v, hi, lo);
  packed[idx] = hi;
  packed[(int64_t)rows * kpad + idx] = lo;
}

int tc_pack_istft(const float* kc, const float* ks, int n_fft, int f_in, int onesided, void* packed,
                  cudaStream_t stream, int transposed) {
  tc_forget_packed(packed);
  const int bn = tc_istft_bn(n_fft);
  const int rows = (n_fft + bn - 1) / bn * bn;
  const int kpad = tc_istft_k(f_in);
  const int64_t n = (int64_t)rows * kpad;
  pack_istft_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, stream>>>(
      kc, ks, n_fft, f_in, onesided, transposed, rows, kpad, (__nv_bfloat16*)packed);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

size_t tc_istft_planes_bytes(int64_t B, int64_t T, int f_in) {
  const int kpad = tc_istft_k(f_in);
  return tc_workspace_bytes(B, T * kpad, kpad, kpad, 0);
}

// X (B, F, T, 2) fp32 -> A planes: row g = b*T + t, column part*F + f (K-major), bf16 hi/lo.
// LANES (inverse STFT pools): plane row b*T + t comes from X[lanes[b].row, :, t] of (R, F, x_T, 2) frames for
// t < lanes[b].T, and is zeros past it and for row -1 (frames past a lane's count are never read: NaN * 0 is NaN).
template <bool LANES>
__global__ void __launch_bounds__(256) istft_prep_kernel(const float* __restrict__ X, int f_in,
                                                         int64_t T, int kpad, int64_t plane_stride,
                                                         __nv_bfloat16* __restrict__ planes,
                                                         const nnab_istft_lane* __restrict__ lanes, int64_t x_T) {
  __shared__ float tile[2][32][33];
  const int64_t b = blockIdx.z;
  const int64_t t0 = (int64_t)blockIdx.x * 32;
  const int f0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const float* __restrict__ Xb = X + b * (int64_t)f_in * T * 2;
  int64_t t_read = T;  // frames of this row that X holds
  if constexpr (LANES) {
    const int64_t row = lanes[b].row;
    t_read = row >= 0 ? lanes[b].T : 0;
    Xb = X + (row >= 0 ? row : 0) * (int64_t)f_in * x_T * 2;
  } else {
    x_T = T;
  }
  for (int r = ty; r < 32; r += 8) {
    const int f = f0 + r;
    const int64_t t = t0 + tx;
    float2 v = make_float2(0.f, 0.f);
    if (f < f_in && t < t_read) v = *reinterpret_cast<const float2*>(Xb + ((int64_t)f * x_T + t) * 2);
    tile[0][r][tx] = v.x;
    tile[1][r][tx] = v.y;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int64_t t = t0 + r;
    const int f = f0 + tx;
    if (t < T && f < f_in) {
      const int64_t row = (b * T + t) * kpad;
#pragma unroll
      for (int part = 0; part < 2; ++part) {
        __nv_bfloat16 hi, lo;
        split_bf16(tile[part][tx][r], hi, lo);
        planes[row + part * f_in + f] = hi;
        planes[plane_stride + row + part * f_in + f] = lo;
      }
    }
  }
}

// The A planes of B x T frames: zeroed where istft_prep_kernel writes nothing, then that kernel's launch.
static int launch_istft_prep(const float* X, int64_t B, int f_in, int64_t T, void* planes_v,
                             const nnab_istft_lane* lanes, int64_t x_T, cudaStream_t stream) {
  if (B > 65535) return NNAB_EUNSUPPORTED;
  const int kpad = tc_istft_k(f_in);
  const SplitGeom g = split_geom(B, T * kpad, kpad, kpad, 0);
  __nv_bfloat16* planes = (__nv_bfloat16*)planes_v;
  // zero everything once when K has padding columns, else just the overhang rows
  if (kpad != 2 * f_in) {
    NNAB_CUDA_TRY(cudaMemsetAsync(planes, 0, (size_t)2 * g.plane_stride * sizeof(__nv_bfloat16), stream));
  } else {
    const int rc = zero_tail(planes, g.nv * kpad, g.plane_stride, stream);
    if (rc) return rc;
  }
  dim3 grid((unsigned)ceil_div64(T, 32), (unsigned)((f_in + 31) / 32), (unsigned)B);
  if (lanes != nullptr)
    istft_prep_kernel<true><<<grid, 256, 0, stream>>>(X, f_in, T, kpad, g.plane_stride, planes, lanes, x_T);
  else
    istft_prep_kernel<false><<<grid, 256, 0, stream>>>(X, f_in, T, kpad, g.plane_stride, planes, nullptr, T);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

int tc_istft_prep(const float* X, int64_t B, int f_in, int64_t T, void* planes_v,
                  cudaStream_t stream) {
  return launch_istft_prep(X, B, f_in, T, planes_v, nullptr, T, stream);
}

int tc_istft_pool_prep(const float* X, const nnab_istft_lane* lanes, int64_t n_lanes, int f_in, int64_t T_max,
                       int64_t x_T, void* planes, cudaStream_t stream) {
  return launch_istft_prep(X, n_lanes, f_in, T_max, planes, lanes, x_T, stream);
}

// ---------------------------------------------------------------------------
// Weight gradient dW[m, k] = sum_{b,t} G[m, (b,t)] * frame_{b,t}[k]   (m = re rows then im rows)
// as a GEMM on the same kernel: the gradient rows are the "signal" (plain-matrix rows of
// length G = B*T), the transposed frame matrix FT[k][(b,t)] takes the packed-basis slot.
// ---------------------------------------------------------------------------
int64_t tc_dw_gpad(int64_t B, int64_t T) { return (B * T + 63) / 64 * 64; }

size_t tc_dw_grad_planes_bytes(int64_t B, int64_t T, int F) {
  const int64_t gpad = tc_dw_gpad(B, T);
  return tc_workspace_bytes(1, (int64_t)2 * F * gpad, (int)gpad, (int)gpad, 0);
}
size_t tc_dw_frames_bytes(int64_t B, int64_t T, int K) {
  const int bn = tc_istft_bn(K);
  const size_t rows = (size_t)((K + bn - 1) / bn) * bn;
  return 2 * rows * (size_t)tc_dw_gpad(B, T) * sizeof(__nv_bfloat16) + 256;
}

// g (B, F, T, 2) -> rows part*F + f, columns b*T + t (bf16 hi/lo planes)
__global__ void __launch_bounds__(256) dw_prep_grad_kernel(const float* __restrict__ g, int F,
                                                           int64_t T, int64_t gpad,
                                                           int64_t plane_stride,
                                                           __nv_bfloat16* __restrict__ planes) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int f = blockIdx.y;
  const int64_t b = blockIdx.z;
  if (t >= T) return;
  const float2 v = *reinterpret_cast<const float2*>(g + (((int64_t)b * F + f) * T + t) * 2);
  const int64_t col = b * T + t;
  __nv_bfloat16 hi, lo;
  split_bf16(v.x, hi, lo);
  planes[(int64_t)f * gpad + col] = hi;
  planes[plane_stride + (int64_t)f * gpad + col] = lo;
  split_bf16(v.y, hi, lo);
  planes[(int64_t)(F + f) * gpad + col] = hi;
  planes[plane_stride + (int64_t)(F + f) * gpad + col] = lo;
}

int tc_dw_prep_grad(const float* g, int64_t B, int F, int64_t T, void* planes_v, cudaStream_t stream) {
  if (B > 65535 || F > 65535) return NNAB_EUNSUPPORTED;
  const int64_t gpad = tc_dw_gpad(B, T);
  const SplitGeom geo = split_geom(1, (int64_t)2 * F * gpad, (int)gpad, (int)gpad, 0);
  __nv_bfloat16* planes = (__nv_bfloat16*)planes_v;
  NNAB_CUDA_TRY(cudaMemsetAsync(planes, 0, (size_t)2 * geo.plane_stride * sizeof(__nv_bfloat16), stream));
  dim3 grid((unsigned)ceil_div64(T, 256), (unsigned)F, (unsigned)B);
  dw_prep_grad_kernel<<<grid, 256, 0, stream>>>(g, F, T, gpad, geo.plane_stride, planes);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

// FT[k][b*T + t] = xpad[b, t*hop + k]   (packed-basis layout: [plane][rows][gpad])
__global__ void __launch_bounds__(256) dw_prep_frames_kernel(
    const float* __restrict__ x, int64_t L, int64_t x_pitch, int K, int hop, int pad, int pad_mode,
    int64_t T, int64_t G, int64_t gpad, int64_t rows, __nv_bfloat16* __restrict__ packed) {
  __shared__ float tile[32][33];
  const int64_t c0 = (int64_t)blockIdx.x * 32;
  const int k0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int r = ty; r < 32; r += 8) {  // r: column (frame) index in the tile, tx: k
    const int64_t c = c0 + r;
    const int k = k0 + tx;
    float v = 0.f;
    if (c < G && k < K) {
      const int64_t b = c / T, t = c - b * T;
      int64_t j = t * hop + k - pad;
      if (j < 0) j = (pad_mode == NNAB_PAD_REFLECT) ? -j : -1;
      else if (j >= L) j = (pad_mode == NNAB_PAD_REFLECT) ? 2 * (L - 1) - j : -1;
      if (j >= 0 && j < L) v = __ldg(x + b * x_pitch + j);
    }
    tile[r][tx] = v;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {  // r: k index in the tile, tx: frame
    const int k = k0 + r;
    const int64_t c = c0 + tx;
    if (k < K && c < G) {
      __nv_bfloat16 hi, lo;
      split_bf16(tile[tx][r], hi, lo);
      packed[(int64_t)k * gpad + c] = hi;
      packed[rows * gpad + (int64_t)k * gpad + c] = lo;
    }
  }
}

int tc_dw_prep_frames(const float* x, int64_t B, int64_t L, int64_t x_pitch, int K, int hop, int pad,
                      int pad_mode, int64_t T, void* packed_v, cudaStream_t stream) {
  const int64_t G = B * T, gpad = tc_dw_gpad(B, T);
  const int bn = tc_istft_bn(K);
  const int64_t rows = (int64_t)((K + bn - 1) / bn) * bn;
  __nv_bfloat16* packed = (__nv_bfloat16*)packed_v;
  tc_forget_packed(packed_v);
  NNAB_CUDA_TRY(cudaMemsetAsync(packed, 0, (size_t)2 * rows * gpad * sizeof(__nv_bfloat16), stream));
  if ((K + 31) / 32 > 65535) return NNAB_EUNSUPPORTED;
  dim3 grid((unsigned)ceil_div64(G, 32), (unsigned)((K + 31) / 32));
  dw_prep_frames_kernel<<<grid, 256, 0, stream>>>(x, L, x_pitch, K, hop, pad, pad_mode, T, G, gpad,
                                                  rows, packed);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

// Adjoint of nn.ReflectionPad1d / ConstantPad1d(pad): fold the gradient of the padded signal
// back onto the clip (mirror margins add onto samples 1..pad and L-1-pad..L-2).
__global__ void __launch_bounds__(256) unpad_adjoint_kernel(const float* __restrict__ gp,
                                                            int64_t gp_pitch, int64_t gp_len,
                                                            int pad, int pad_mode, int64_t L,
                                                            float* __restrict__ dx) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t b = blockIdx.y;
  if (j >= L) return;
  const float* __restrict__ g = gp + b * gp_pitch;
  auto at = [&](int64_t i) { return (i >= 0 && i < gp_len) ? g[i] : 0.f; };
  float v = at(pad + j);
  if (pad > 0 && pad_mode == NNAB_PAD_REFLECT) {
    if (j >= 1 && j <= pad) v += at(pad - j);
    if (j >= L - 1 - pad && j <= L - 2) v += at(pad + 2 * (L - 1) - j);
  }
  dx[b * L + j] = v;
}

int tc_unpad_adjoint(const float* gp, int64_t gp_pitch, int64_t gp_len, int64_t B, int pad,
                     int pad_mode, int64_t L, float* dx, cudaStream_t stream) {
  if (B > 65535) return NNAB_EUNSUPPORTED;
  if (B <= 0 || L <= 0) return NNAB_OK;
  dim3 grid((unsigned)ceil_div64(L, 256), (unsigned)B);
  unpad_adjoint_kernel<<<grid, 256, 0, stream>>>(gp, gp_pitch, gp_len, pad, pad_mode, L, dx);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

// Window sum-square of overlap-add position s over T frames (utils.py:43-49), summed from the last frame that
// covers s down: the one order every inverse-STFT finalize uses.
__device__ __forceinline__ float istft_wss(const float* __restrict__ window, int n_fft, int hop, int64_t T,
                                           int64_t s) {
  int64_t t_hi = s / hop;
  if (t_hi > T - 1) t_hi = T - 1;
  float wss = 0.f;
  for (int64_t t = t_hi; t >= 0; --t) {
    const int64_t n = s - t * hop;
    if (n >= n_fft) break;
    const float w = __ldg(window + n);
    wss = fmaf(w, w, wss);
  }
  return wss;
}

// Divide the overlap-added frames by the window sum-square (utils.py:43-49; only where it
// exceeds 1e-10) and strip the centre padding: out[b, i] = ola[b, i + offset] / wss(i + offset).
__global__ void __launch_bounds__(256) istft_finalize_kernel(const float* __restrict__ ola,
                                                             int64_t ola_pitch,
                                                             const float* __restrict__ window,
                                                             int n_fft, int hop, int64_t T,
                                                             int64_t offset, float* __restrict__ out,
                                                             int64_t out_len) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t b = blockIdx.y;
  if (i >= out_len) return;
  const int64_t s = i + offset;
  const float wss = istft_wss(window, n_fft, hop, T, s);
  float v = ola[b * ola_pitch + s];
  if (wss > 1e-10f) v = v / wss;
  out[b * out_len + i] = v;
}

int tc_istft_finalize(const float* ola, int64_t ola_pitch, int64_t B, const float* window,
                      int n_fft, int hop, int64_t T, int64_t offset, float* out, int64_t out_len,
                      cudaStream_t stream) {
  if (B > 65535) return NNAB_EUNSUPPORTED;
  if (out_len <= 0 || B <= 0) return NNAB_OK;
  dim3 grid((unsigned)ceil_div64(out_len, 256), (unsigned)B);
  istft_finalize_kernel<<<grid, 256, 0, stream>>>(ola, ola_pitch, window, n_fft, hop, T, offset,
                                                  out, out_len);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

// Streamed inverse STFT pushes.  Lane i is lanes[i] of the DEVICE lane table or, without one (a lock-step push
// of B streams that share their counters), `shared` in slot i.  Row i of the overlap-add buffer holds lane i's
// global positions from frames_i * hop - lead on (lead = n_fft): its carried sums start at most hop - n_fft / 2
// positions before frames_i * hop (istft_chunk_plan's origin), so every lane's new frames start at column `lead`
// and one FMT_OLA GEMM with out = ola + lead serves all rows.  The seed writes each row whole: the lane's carried
// sums from state row slot_i where they lie, zeros elsewhere.
__global__ void __launch_bounds__(256) istft_pool_seed_kernel(const nnab_istft_lane* __restrict__ lanes,
                                                              const nnab_istft_lane shared,
                                                              const float* __restrict__ state, int n_fft,
                                                              int hop, int center, int64_t lead,
                                                              float* __restrict__ ola, int64_t ola_pitch) {
  nnab_istft_lane ln = shared;
  ln.slot = blockIdx.y;
  if (lanes != nullptr) ln = lanes[blockIdx.y];
  const IstftChunkPlan pl = istft_lane_plan(ln, n_fft, hop, center);
  const int64_t base = ln.frames * hop - lead - pl.origin;  // column c holds carried position c + base
  const float* __restrict__ src = state + ln.slot * n_fft;
  float* __restrict__ row = ola + (int64_t)blockIdx.y * ola_pitch;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < ola_pitch;
       c += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = c + base;
    row[c] = k >= 0 && k < pl.carried ? __ldg(src + k) : 0.f;
  }
}

// Rows i < A of out (A, n_max) take lane i's final samples, each divided by the window sum-square of its global
// position over the lane's frames_i + T_i frames (istft_wss: the same sum, in the same order, as
// istft_finalize_kernel), then exact zeros up to n_max; every lane's open tail goes un-normalised to its state row.
__global__ void __launch_bounds__(256) istft_pool_finalize_kernel(
    const nnab_istft_lane* __restrict__ lanes, const nnab_istft_lane shared, int64_t A,
    const float* __restrict__ ola, int64_t ola_pitch, int64_t lead, const float* __restrict__ window, int n_fft,
    int hop, int center, float* __restrict__ out, int64_t n_max, float* __restrict__ state) {
  const int64_t i = blockIdx.y;
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  nnab_istft_lane ln = shared;
  ln.slot = i;
  if (lanes != nullptr) ln = lanes[i];
  const IstftChunkPlan pl = istft_lane_plan(ln, n_fft, hop, center);
  const float* __restrict__ row = ola + i * ola_pitch;
  const int64_t base = ln.frames * hop - lead;  // global position of column 0
  if (i < A && j < n_max) {
    float v = 0.f;
    if (j < pl.emit_end - pl.emit_begin) {
      const int64_t s = pl.emit_begin + j;
      const float wss = istft_wss(window, n_fft, hop, ln.frames + ln.T, s);
      v = row[s - base];
      if (wss > 1e-10f) v = v / wss;
    }
    out[i * n_max + j] = v;
  }
  if (j < pl.carry_len) state[ln.slot * n_fft + j] = row[pl.carry_begin - base + j];
}

int tc_istft_pool_seed(const nnab_istft_lane* lanes, const nnab_istft_lane& shared, int64_t n_lanes,
                       const float* state, int n_fft, int hop, int center, int64_t lead, float* ola, int64_t ola_pitch,
                       cudaStream_t stream) {
  if (n_lanes > 65535) return NNAB_EUNSUPPORTED;
  if (n_lanes <= 0) return NNAB_OK;
  const dim3 grid((unsigned)ceil_div64(ola_pitch, 256), (unsigned)n_lanes);
  istft_pool_seed_kernel<<<grid, 256, 0, stream>>>(lanes, shared, state, n_fft, hop, center, lead, ola, ola_pitch);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

int tc_istft_pool_finalize(const nnab_istft_lane* lanes, const nnab_istft_lane& shared, int64_t n_lanes, int64_t A,
                           const float* ola, int64_t ola_pitch, int64_t lead, const float* window, int n_fft, int hop,
                           int center, float* out, int64_t n_max, float* state, cudaStream_t stream) {
  if (n_lanes > 65535) return NNAB_EUNSUPPORTED;
  if (n_lanes <= 0) return NNAB_OK;
  const int64_t n = n_max > n_fft ? n_max : n_fft;  // a carried tail holds at most n_fft positions
  const dim3 grid((unsigned)ceil_div64(n, 256), (unsigned)n_lanes);
  istft_pool_finalize_kernel<<<grid, 256, 0, stream>>>(lanes, shared, A, ola, ola_pitch, lead, window, n_fft, hop,
                                                       center, out, n_max, state);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

// PTX wrappers: tc_ptx.cuh

// ---------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------
struct TcParams {
  int num_m_tiles, num_n_tiles, bn;
  int rows_mode;   // 1: A viewed as (rows x hop) matrix (BK | hop); 0: overlapping-stride map
  int hop;          // effective hop (hop * phases)
  int t_mul, t_add;  // output frame index = t * t_mul + t_add (frame phases)
  int k_splits;      // >1: every (m, n) tile is cut into k_splits K-chunks (FMT_RAW epilogue)
  int64_t nv, t_slots, T;  // T = valid frames of this phase
  int kb_begin[TC_MAX_N_TILES];
  int kb_end[TC_MAX_N_TILES];
  EpiParams epi;
};

// Work order of a persistent worker: its u-th unit (unit = tile * ks + K-chunk), or -1 when done.
// Split-K partial sums are combined by ORDERED read-modify-writes (run-to-run identical; no atomics,
// no zero-fill of the scratch): all chunks of a tile go to the same worker, consecutively, so chunk c
// of a tile adds after chunk c-1 has stored, in program order of one thread.  (A balanced round-robin
// of the units with flag-ordered adds measured 2.04 ms vs 1.27 ms at cfg3: the chunks of a tile
// finish their MMAs together and their epilogues then serialise.)
__device__ __forceinline__ int sched_tile(int u, int worker, int n_workers, int num_mn, int ks) {
  const int mn = worker + (u / ks) * n_workers;
  return mn < num_mn ? mn * ks + (u % ks) : -1;
}

// tile index -> (m tile, n tile, k-block range); K-chunks of one (m, n) tile are adjacent
__device__ __forceinline__ void decode_tile(const TcParams& p, int tile, int& m_tile, int& n_tile,
                                            int& kb0, int& kb1) {
  const int ks = tile % p.k_splits;
  const int mn = tile / p.k_splits;
  m_tile = mn / p.num_n_tiles;
  n_tile = mn - m_tile * p.num_n_tiles;
  const int lo = p.kb_begin[n_tile], n = p.kb_end[n_tile] - lo;
  kb0 = lo + (int)(((int64_t)n * ks) / p.k_splits);
  kb1 = lo + (int)(((int64_t)n * (ks + 1)) / p.k_splits);
}

// Read one 128-frame x bn accumulator tile out of shared memory (this warp's 32 lanes =
// 32 consecutive frames) and emit it in the requested output format.
template <int FMT>
__device__ __forceinline__ void epilogue_tile(const TcParams& p, uint32_t trow, int64_t g,
                                              int n_tile, int half, int k_chunk, int mn_tile) {
      const int64_t b = g / p.t_slots;
      const int64_t tl = g - b * p.t_slots;
      const bool valid = (g < p.nv) && (tl < p.T);
      const int64_t t = tl * p.t_mul + p.t_add;  // frame index in the output
      const int f_base = n_tile * half;
      if constexpr (FMT == 8) {
        // ---- inverse STFT: window the frame's samples and overlap-add them ----
        float* dst = p.epi.out + b * p.epi.ola_pitch + t * p.epi.ola_hop;
        const int n_base = n_tile * (2 * half);
#pragma unroll 1
        for (int c0 = 0; c0 < 2 * half; c0 += 8) {
          uint32_t v[8];
          acc_ld8(trow + (uint32_t)c0, v);
          if (valid) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int n = n_base + c0 + j;
              if (n < p.epi.F)  // F = n_fft samples per frame
                atomicAdd(dst + n, p.epi.scale != nullptr
                                       ? __uint_as_float(v[j]) * __ldg(p.epi.scale + n)
                                       : __uint_as_float(v[j]));
            }
          }
        }
      } else if constexpr (FMT == 7) {
        // ---- split-K partial sums: ordered read-modify-write of the raw planes (this thread owns
        // the element for every chunk of the tile; chunk 0 stores, later chunks add) ----
        float* rre = p.epi.raw + ((int64_t)b * p.epi.F) * p.epi.T + t;
#pragma unroll 1
        for (int c0 = 0; c0 < half; c0 += 8) {
          uint32_t re[8], im[8];
          acc_ld8(trow + (uint32_t)c0, re);
          acc_ld8(trow + (uint32_t)(half + c0), im);
          if (valid) {
            const int jmax = min(8, min(half - c0, p.epi.F - f_base - c0));
#pragma unroll
            for (int j = 0; j < 8; ++j)
              if (j < jmax) {
                float* q = rre + (int64_t)(f_base + c0 + j) * p.epi.T;
                float vr = __uint_as_float(re[j]), vi = __uint_as_float(im[j]);
                if (k_chunk > 0) { vr += __ldcg(q); vi += __ldcg(q + p.epi.raw_plane); }
                __stcg(q, vr);
                __stcg(q + p.epi.raw_plane, vi);
              }
          }
        }

      } else if constexpr (FMT == 6) {
        // ---- FIR decimator stage: this thread holds outputs n0 .. n0 + 2*half - 1 of clip b ----
        epilogue_decim(p.epi.dec, trow, b, tl, valid, half);
      } else if constexpr (FMT == 5) {
        // ---- fused banded filterbank: two running filter sums per frame ----
        float* mel = p.epi.out + ((int64_t)b * p.epi.n_fb) * p.epi.T + t;
        int cj0 = -1, cj1 = -1;
        float a0 = 0.f, a1 = 0.f;
        // rolled loop over 8-column loads: the body must stay I-cache resident
        // (a 32x unrolled version was ~80 KB of code per tile and fetch-stalled)
#pragma unroll 1
        for (int c0 = 0; c0 < half; c0 += 8) {
          uint32_t re[8], im[8];
          acc_ld8(trow + (uint32_t)c0, re);
          acc_ld8(trow + (uint32_t)(half + c0), im);
          const int jmax = min(8, min(half - c0, p.epi.F - f_base - c0));
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if (j < jmax) {  // warp-uniform
              const int4 raw = __ldg(reinterpret_cast<const int4*>(p.epi.fb_table) + f_base + c0 + j);
              const float pw = epi_power(p.epi, __uint_as_float(re[j]), __uint_as_float(im[j]));
              if (raw.x != cj0) {
                if (raw.x == cj1) {
                  const int tj = cj0; cj0 = cj1; cj1 = tj;
                  const float ta = a0; a0 = a1; a1 = ta;
                } else {
                  if (cj0 >= 0 && valid) atomicAdd(mel + (int64_t)cj0 * p.epi.T, a0);
                  cj0 = raw.x; a0 = 0.f;
                }
              }
              if (raw.y != cj1) {
                if (cj1 >= 0 && valid) atomicAdd(mel + (int64_t)cj1 * p.epi.T, a1);
                cj1 = raw.y; a1 = 0.f;
              }
              a0 = fmaf(__int_as_float(raw.z), pw, a0);
              a1 = fmaf(__int_as_float(raw.w), pw, a1);
            }
          }
        }
        if (cj0 >= 0 && valid) atomicAdd(mel + (int64_t)cj0 * p.epi.T, a0);
        if (cj1 >= 0 && valid) atomicAdd(mel + (int64_t)cj1 * p.epi.T, a1);
      } else {
      constexpr int CH = (FMT == NNAB_FMT_COMPLEX || FMT == NNAB_FMT_PHASE_UNIT) ? 2 : 1;
      float* dst = p.epi.out + (((int64_t)b * p.epi.out_bins + p.epi.bin_offset) * p.epi.T + t) * CH;
      if constexpr (FMT == NNAB_FMT_MAGNITUDE || FMT == NNAB_FMT_COMPLEX) {
        // light per-bin code: 32 columns per load, fully unrolled
        for (int c0 = 0; c0 < half; c0 += 32) {
          uint32_t re[32], im[32];
          acc_ld32(trow + (uint32_t)c0, re);
          acc_ld32(trow + (uint32_t)(half + c0), im);
          if (valid) {
            const int jmax = min(32, min(half - c0, p.epi.F - f_base - c0));
            if (jmax == 32) {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                epi_store_fmt<FMT>(p.epi, dst, f_base + c0 + j, __uint_as_float(re[j]),
                                   __uint_as_float(im[j]));
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (j < jmax)
                  epi_store_fmt<FMT>(p.epi, dst, f_base + c0 + j, __uint_as_float(re[j]),
                                     __uint_as_float(im[j]));
            }
          }
        }
      } else {
        // atan2f / sincosf / powf bodies: rolled loop over 8 columns keeps the code I-cache sized
#pragma unroll 1
        for (int c0 = 0; c0 < half; c0 += 8) {
          uint32_t re[8], im[8];
          acc_ld8(trow + (uint32_t)c0, re);
          acc_ld8(trow + (uint32_t)(half + c0), im);
          if (valid) {
            const int jmax = min(8, min(half - c0, p.epi.F - f_base - c0));
#pragma unroll
            for (int j = 0; j < 8; ++j)
              if (j < jmax)
                epi_store_fmt<FMT>(p.epi, dst, f_base + c0 + j, __uint_as_float(re[j]),
                                   __uint_as_float(im[j]));
          }
        }
      }
      }
}

struct TcSmem {
  static constexpr int STAGES = 2;
  static constexpr uint32_t A_BYTES = TC_BM * 64 * 2;   // one plane, 128 rows x 64 bf16
  static constexpr uint32_t B_BYTES = 256 * 64 * 2;     // one plane, <= 256 basis rows
  static constexpr uint32_t STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
  static constexpr uint32_t BAR_OFFSET = STAGES * STAGE_BYTES;
  static constexpr uint32_t TOTAL = BAR_OFFSET + 256 + 1024;  // + barriers + align slack
  // the accumulator tile (128 rows x <= 256 fp32) reuses the stages once a unit's K range is drained
  static_assert(TC_BM * 256 * 4 <= BAR_OFFSET, "accumulator tile does not fit the stage ring");
};

// Persistent over work units (output tile x K chunk).  Per unit the producer streams the K blocks through
// a 2-stage ring, both consumer warpgroups accumulate their 64 rows in registers, then store them into the
// accumulator tile (over the drained ring) and warps 0-3 run the epilogue, one tile row per thread.  The
// producer starts the next unit's loads once the tile has been read out (drained_bar).
template <int FMT>
__global__ void __launch_bounds__(TC_KERNEL_THREADS, 1)
framed_tc_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                 const TcParams p) {
  using S = TcSmem;
  constexpr int BK = 64, STAGES = S::STAGES;
  const uint32_t base = acc_tile_base();
  const uint32_t bar_base = base + S::BAR_OFFSET;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  const uint32_t drained_bar = bar_base + 8u * (2 * STAGES);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);  // one arrival per consumer warp
    }
    mbar_init(drained_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  const int num_mn = p.num_m_tiles * p.num_n_tiles;
  if (warp == TC_PRODUCER_WARP) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      prefetch_tmap(&tm_a);
      prefetch_tmap(&tm_b);
      const uint32_t b_tile_bytes = (uint32_t)p.bn * BK * 2;
      int stage = 0;
      uint32_t phase = 0;
      for (int u = 0, tile; (tile = sched_tile(u, blockIdx.x, gridDim.x, num_mn, p.k_splits)) >= 0; ++u) {
        if (u > 0) mbar_wait(drained_bar, (uint32_t)(u - 1) & 1u);
        int m_tile, n_tile, kb0, kb1;
        decode_tile(p, tile, m_tile, n_tile, kb0, kb1);
        const int m0 = m_tile * TC_BM;
        const int n0 = n_tile * p.bn;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t sb = base + stage * S::STAGE_BYTES;
          mbar_expect_tx(full_bar(stage), 2 * S::A_BYTES + 2 * b_tile_bytes);
          const int k0 = kb * BK;
          int c0 = k0, c1 = m0;
          if (p.rows_mode) {
            c1 = m0 + k0 / p.hop;
            c0 = k0 - (k0 / p.hop) * p.hop;
          }
          tma_load_3d(sb, &tm_a, full_bar(stage), c0, c1, 0);
          tma_load_3d(sb + S::A_BYTES, &tm_a, full_bar(stage), c0, c1, 1);
          tma_load_3d(sb + 2 * S::A_BYTES, &tm_b, full_bar(stage), k0, n0, 0);
          tma_load_3d(sb + 2 * S::A_BYTES + S::B_BYTES, &tm_b, full_bar(stage), k0, n0, 1);
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  // ===================== consumers: wgmma (warpgroup wg = rows 64 wg ..) + epilogue =====================
  const int wg = warp >> 2;
  const uint32_t a_off = (uint32_t)wg * 64u * (BK * 2);
  // Row stride of the accumulator tile: the 32-column read-out of epilogue_tile (Magnitude / Complex)
  // reads im columns half + [0, round_up(half, 32)), past bn when 32 does not divide half; those reads
  // must stay inside the thread's own row (their values are dropped by the jmax guard).
  const int half_n = p.bn >> 1;
  const uint32_t tile_addr = acc_tile(half_n + ((half_n + 31) & ~31));
  float acc[128];
  int stage = 0;
  uint32_t phase = 0;
  for (int u = 0, tile; (tile = sched_tile(u, blockIdx.x, gridDim.x, num_mn, p.k_splits)) >= 0; ++u) {
    int m_tile, n_tile, kb0, kb1;
    decode_tile(p, tile, m_tile, n_tile, kb0, kb1);
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;  // (the previous unit's values are dead after acc_store)
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t sb = base + stage * S::STAGE_BYTES;
      wgmma_fence();
      wg_kblock_split3<256>(p.bn, acc, wg_desc_lo(sb + a_off), wg_desc_lo(sb + S::A_BYTES + a_off),
                            wg_desc_lo(sb + 2 * S::A_BYTES), wg_desc_lo(sb + 2 * S::A_BYTES + S::B_BYTES),
                            kb != kb0);
      wgmma_commit();
      wgmma_wait_all();
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(stage));  // this warp is done reading the stage
      if (++stage == STAGES) { stage = 0; phase ^= 1u; }
    }
    consumer_sync();  // both warpgroups are done with the ring: the tile may overwrite it
    acc_store<256>(tile_addr, acc, p.bn, wg * 64);
    consumer_sync();
    if (warp < 4) {
      const int64_t g = (int64_t)m_tile * TC_BM + warp * 32 + lane;
      epilogue_tile<FMT>(p, tile_addr + acc_row((uint32_t)warp * 32u), g, n_tile, p.bn >> 1,
                         tile % p.k_splits, tile / p.k_splits);
    }
    fence_proxy_async();  // the next TMA writes land on bytes the tile occupied
    consumer_sync();
    if (threadIdx.x == 0) mbar_arrive(drained_bar);
  }
}


// ===========================================================================
// Per-K-block MMA width for banks
// whose rows have nested, centred supports (CQT1992v2).
//
// Packed rows are ordered in 8-bin groups, [re bins 8g..8g+7 | negated im of the same bins], so
// basis row r is accumulator column r and a K block that only the G longest groups reach needs
// an MMA of width N = 16 G: TMA fetches 16 G basis rows, the wgmma instruction is the one of width N,
// the accumulation still lands in accumulator columns [0, N).  K blocks are visited in order
// of decreasing width, so the first MMA of a tile (accumulate = 0) initialises every column the
// tile will touch, and the epilogue of a split-K chunk reads only those.
// ===========================================================================
constexpr int VN_MAX_BLOCKS = 512;
struct VarNPlan {
  int n_blocks;              // active K blocks
  int n_chunks;              // split-K chunks (1 = none)
  int chunk_begin[17];       // chunk c = ordered blocks [chunk_begin[c], chunk_begin[c+1])
  uint16_t order[VN_MAX_BLOCKS];  // K block index (64 samples each), widest first
  uint8_t groups[VN_MAX_BLOCKS];  // 8-bin groups the block reaches (N = 16 * groups)
};

// packed[plane][row][k]: row = 16 g + 8 part + j  <->  bin 8 g + j, part 0 = re, 1 = negated im
__global__ void __launch_bounds__(256) pack_basis_varn_kernel(
    const float* __restrict__ w_re, const float* __restrict__ w_im, int F, int K, int rows, int kpad,
    __nv_bfloat16* __restrict__ packed) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int k8 = kpad / 8;
  if (idx >= (int64_t)rows * k8) return;
  const int r = (int)(idx / k8);
  const int k0 = (int)(idx % k8) * 8;
  const int f = (r >> 4) * 8 + (r & 7);
  const int part = (r >> 3) & 1;
  __align__(16) __nv_bfloat16 hi[8];
  __align__(16) __nv_bfloat16 lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = k0 + e;
    float v = 0.f;
    if (f < F && k < K)
      v = part == 0 ? __ldg(w_re + (int64_t)f * K + k) : -__ldg(w_im + (int64_t)f * K + k);
    split_bf16(v, hi[e], lo[e]);
  }
  const int64_t o = (int64_t)r * kpad + k0;
  *reinterpret_cast<uint4*>(packed + o) = *reinterpret_cast<const uint4*>(hi);
  *reinterpret_cast<uint4*>(packed + (int64_t)rows * kpad + o) = *reinterpret_cast<const uint4*>(lo);
}

// FMT: 0 Magnitude, 1 Complex, 3 PhaseUnit (direct), 7 split-K partial sums.
template <int FMT>
__device__ __forceinline__ void epilogue_tile_varn(const TcParams& p, uint32_t trow, int64_t g,
                                                   int n_groups, int k_chunk, int mn_tile) {
  const int64_t b = g / p.t_slots;
  const int64_t tl = g - b * p.t_slots;
  const bool valid = (g < p.nv) && (tl < p.T);
  const int64_t t = tl * p.t_mul + p.t_add;
  constexpr int CH = (FMT == NNAB_FMT_COMPLEX || FMT == NNAB_FMT_PHASE_UNIT) ? 2 : 1;
  float* dst = p.epi.out + (((int64_t)b * p.epi.out_bins + p.epi.bin_offset) * p.epi.T + t) * CH;
  float* rre = (FMT == 7) ? p.epi.raw + ((int64_t)b * p.epi.F) * p.epi.T + t : nullptr;
#pragma unroll 1
  for (int gi = 0; gi < n_groups; ++gi) {
    uint32_t re[8], im[8];
    acc_ld8(trow + (uint32_t)(16 * gi), re);
    acc_ld8(trow + (uint32_t)(16 * gi + 8), im);
    if (valid) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int f = 8 * gi + j;
        if (f < p.epi.F) {
          if constexpr (FMT == 7) {
            float* q = rre + (int64_t)f * p.epi.T;
            float vr = __uint_as_float(re[j]), vi = __uint_as_float(im[j]);
            if (k_chunk > 0) { vr += __ldcg(q); vi += __ldcg(q + p.epi.raw_plane); }  // ordered by chunk
            __stcg(q, vr);
            __stcg(q + p.epi.raw_plane, vi);
          } else {
            epi_store_fmt<FMT>(p.epi, dst, f, __uint_as_float(re[j]), __uint_as_float(im[j]));
          }
        }
      }
    }
  }
}

template <int FMT>
__global__ void __launch_bounds__(TC_KERNEL_THREADS, 1)
framed_tcv_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b8,
                  const __grid_constant__ CUtensorMap tm_b32, const TcParams p,
                  const __grid_constant__ VarNPlan plan) {
  using S = TcSmem;
  constexpr int BK = 64, STAGES = S::STAGES;
  const uint32_t base = acc_tile_base();
  const uint32_t bar_base = base + S::BAR_OFFSET;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  const uint32_t drained_bar = bar_base + 8u * (2 * STAGES);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);
    }
    mbar_init(drained_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == TC_PRODUCER_WARP) {
    if (elect_one()) {
      prefetch_tmap(&tm_a);
      prefetch_tmap(&tm_b8);
      prefetch_tmap(&tm_b32);
      int stage = 0;
      uint32_t phase = 0;
      for (int u = 0, tile; (tile = sched_tile(u, blockIdx.x, gridDim.x, p.num_m_tiles, plan.n_chunks)) >= 0; ++u) {
        if (u > 0) mbar_wait(drained_bar, (uint32_t)(u - 1) & 1u);
        const int chunk = tile % plan.n_chunks;
        const int m0 = (tile / plan.n_chunks) * TC_BM;
        for (int i = plan.chunk_begin[chunk]; i < plan.chunk_begin[chunk + 1]; ++i) {
          const int k0 = (int)plan.order[i] * BK;
          const int rows = 16 * (int)plan.groups[i];  // basis rows of the block's MMA width
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t sb = base + stage * S::STAGE_BYTES;
          mbar_expect_tx(full_bar(stage), 2 * S::A_BYTES + 2 * (uint32_t)rows * BK * 2);
          int c0 = k0, c1 = m0;
          if (p.rows_mode) {
            c1 = m0 + k0 / p.hop;
            c0 = k0 - (k0 / p.hop) * p.hop;
          }
          tma_load_3d(sb, &tm_a, full_bar(stage), c0, c1, 0);
          tma_load_3d(sb + S::A_BYTES, &tm_a, full_bar(stage), c0, c1, 1);
          const uint32_t bh = sb + 2 * S::A_BYTES, bl = bh + S::B_BYTES;
          int r = 0;
          for (; rows - r >= 32; r += 32) {
            tma_load_3d(bh + (uint32_t)r * BK * 2, &tm_b32, full_bar(stage), k0, r, 0);
            tma_load_3d(bl + (uint32_t)r * BK * 2, &tm_b32, full_bar(stage), k0, r, 1);
          }
          for (; r < rows; r += 8) {
            tma_load_3d(bh + (uint32_t)r * BK * 2, &tm_b8, full_bar(stage), k0, r, 0);
            tma_load_3d(bl + (uint32_t)r * BK * 2, &tm_b8, full_bar(stage), k0, r, 1);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;
  const uint32_t a_off = (uint32_t)wg * 64u * (BK * 2);
  const uint32_t tile_addr = acc_tile(p.bn);
  float acc[128];
  int stage = 0;
  uint32_t phase = 0;
  for (int u = 0, tile; (tile = sched_tile(u, blockIdx.x, gridDim.x, p.num_m_tiles, plan.n_chunks)) >= 0; ++u) {
    const int chunk = tile % plan.n_chunks;
    const int m_tile = tile / plan.n_chunks;
    const int i0 = plan.chunk_begin[chunk];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    for (int i = i0; i < plan.chunk_begin[chunk + 1]; ++i) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t sb = base + stage * S::STAGE_BYTES;
      wgmma_fence();
      wg_kblock_split3<256>(16 * (int)plan.groups[i], acc, wg_desc_lo(sb + a_off),
                            wg_desc_lo(sb + S::A_BYTES + a_off), wg_desc_lo(sb + 2 * S::A_BYTES),
                            wg_desc_lo(sb + 2 * S::A_BYTES + S::B_BYTES), i != i0);
      wgmma_commit();
      wgmma_wait_all();
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(stage));
      if (++stage == STAGES) { stage = 0; phase ^= 1u; }
    }
    // widest block of the chunk = its first: the columns this unit initialised
    const int n_groups = (int)plan.groups[i0];
    consumer_sync();
    acc_store<256>(tile_addr, acc, 16 * n_groups, wg * 64);
    consumer_sync();
    if (warp < 4) {
      const int64_t g = (int64_t)m_tile * TC_BM + warp * 32 + lane;
      epilogue_tile_varn<FMT>(p, tile_addr + acc_row((uint32_t)warp * 32u), g, n_groups, chunk, m_tile);
    }
    fence_proxy_async();
    consumer_sync();
    if (threadIdx.x == 0) mbar_arrive(drained_bar);
  }
}

// Split-K finalize: raw (re, im) sums -> per-bin scale + output format (generic epilogue).
__global__ void __launch_bounds__(256) splitk_finalize_kernel(const EpiParams e, int64_t B) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int f = blockIdx.y;
  if (t >= e.T) return;
  for (int64_t b = blockIdx.z; b < B; b += gridDim.z) {
    const int64_t i = ((int64_t)b * e.F + f) * e.T + t;
    epi_store(e, b, f, t, e.raw[i], e.raw[e.raw_plane + i]);
  }
}

// Long kernels only: the scratch exists to bound the tensor-core accumulation length
// (its error grows with the number of accumulated MMAs) and to even out the tile count.
size_t tc_splitk_scratch_bytes(int64_t B, int F, int64_t T, int K) {
  if (K < 8192) return 0;
  return (size_t)2 * B * F * T * sizeof(float) + 256;
}

// ---------------------------------------------------------------------------
// pre-pass of a streamed push (chunk_split_kernel, chunk_carry_kernel)
// ---------------------------------------------------------------------------
static int launch_chunk_split(const ChunkSource& cs, int x_dtype, dim3 grid, int shift, int64_t clip_pitch,
                              int64_t plane_stride, int poly_hop, __nv_bfloat16* planes, cudaStream_t stream) {
  return with_sample_type(x_dtype, cs.chunk, [&](auto* xs) {
    using Tx = std::remove_const_t<std::remove_pointer_t<decltype(xs)>>;
    if (cs.rows != nullptr)
      chunk_split_rows_kernel<Tx><<<grid, 256, 0, stream>>>(cs, xs, shift, clip_pitch, plane_stride, poly_hop,
                                                            planes);
    else
      chunk_split_kernel<Tx><<<grid, 256, 0, stream>>>(cs, xs, shift, clip_pitch, plane_stride, poly_hop, planes);
  });
}

int tc_chunk_split(const ChunkSource& cs, int x_dtype, int64_t B, int64_t clip_pitch, int64_t plane_stride,
                   void* planes, cudaStream_t stream) {
  if (B <= 0 || clip_pitch <= 0) return NNAB_OK;
  if (B > 65535 || clip_pitch % 8 != 0) return NNAB_EUNSUPPORTED;
  const dim3 grid((unsigned)ceil_div64(clip_pitch, 256 * 8), (unsigned)B);
  return launch_chunk_split(cs, x_dtype, grid, 0, clip_pitch, plane_stride, 0, static_cast<__nv_bfloat16*>(planes),
                            stream);
}

int tc_pool_carry(const ChunkSource& cs, int x_dtype, int64_t n_lanes, int64_t longest, cudaStream_t stream) {
  if (longest <= 0 || n_lanes <= 0) return NNAB_OK;
  if (n_lanes > 65535) return NNAB_EUNSUPPORTED;
  const dim3 grid((unsigned)ceil_div64(longest, 256), (unsigned)n_lanes);
  return with_sample_type(x_dtype, cs.chunk, [&](auto* xs) {
    using Tx = std::remove_const_t<std::remove_pointer_t<decltype(xs)>>;
    chunk_carry_kernel<Tx><<<grid, 256, 0, stream>>>(cs, xs);
  });
}

int tc_pool_mask(const ChunkSource& cs, int64_t A, float* out, int64_t rows, int64_t T, int cols,
                 cudaStream_t stream) {
  if (A <= 0 || T <= 0) return NNAB_OK;
  if (A > 65535) return NNAB_EUNSUPPORTED;
  const int64_t per_row = rows * T * cols;
  const dim3 grid((unsigned)(ceil_div64(per_row, 256) < 64 ? ceil_div64(per_row, 256) : 64), (unsigned)A);
  pool_mask_kernel<<<grid, 256, 0, stream>>>(cs, out, rows, T, cols);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

int tc_pyr_pool_plan(const PyrStream& p, const nnab_stream_lane* lanes, const nnab_stream_lane& shared,
                     int64_t n_lanes, int pad_mode, PyrLaneSig* table, cudaStream_t stream) {
  if (n_lanes <= 0) return NNAB_OK;
  const int64_t n = n_lanes * p.n_sig;
  pyr_pool_plan_kernel<<<(unsigned)ceil_div64(n, 128), 128, 0, stream>>>(p, lanes, shared, n_lanes, pad_mode,
                                                                         table);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

int tc_device_pyramid_plan(const PyrStream& p, int64_t slots, int64_t* counters, const int32_t* lengths,
                           const uint8_t* end, int32_t* errors, int64_t* info, int32_t* counts,
                           nnab_stream_lane* lanes, int64_t chunk, int pad_mode, cudaStream_t stream) {
  device_pyramid_plan_kernel<<<(unsigned)ceil_div64(slots, 128), 128, 0, stream>>>(
      p, slots, counters, lengths, end, errors, info, counts, lanes, chunk, pad_mode);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

int tc_rows_carry(const ChunkSource& cs, int x_dtype, int64_t n_rows, int64_t longest, cudaStream_t stream) {
  if (longest <= 0 || n_rows <= 0) return NNAB_OK;
  if (n_rows > 65535) return NNAB_EUNSUPPORTED;
  const dim3 grid((unsigned)ceil_div64(longest, 256), (unsigned)n_rows);
  return with_sample_type(x_dtype, cs.chunk, [&](auto* xs) {
    using Tx = std::remove_const_t<std::remove_pointer_t<decltype(xs)>>;
    chunk_carry_rows_kernel<Tx><<<grid, 256, 0, stream>>>(cs, xs);
  });
}

int tc_rows_mask(const PyrLaneSig* rows, int64_t A, float* out, int64_t n_rows, int64_t T, int cols,
                 cudaStream_t stream) {
  if (A <= 0 || T <= 0) return NNAB_OK;
  if (A > 65535) return NNAB_EUNSUPPORTED;
  const int64_t per_row = n_rows * T * cols;
  const dim3 grid((unsigned)(ceil_div64(per_row, 256) < 64 ? ceil_div64(per_row, 256) : 64), (unsigned)A);
  rows_mask_kernel<<<grid, 256, 0, stream>>>(rows, out, n_rows, T, cols);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

int encode_3d(CUtensorMap* map, void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                     uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t box0, uint32_t box1,
                     int bk) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) {
    set_error_text("cuTensorMapEncodeTiled entry point not available");
    return NNAB_ECUDA;
  }
  cuuint64_t gdim[3] = {d0, d1, d2};
  cuuint64_t gstr[2] = {stride1_bytes, stride2_bytes};
  cuuint32_t box[3] = {box0, box1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  const CUtensorMapSwizzle sw = (bk == 64) ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, base, gdim, gstr, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[200];
    snprintf(msg, sizeof(msg),
             "cuTensorMapEncodeTiled failed (%d): dims {%llu,%llu,%llu} strides {%llu,%llu} box {%u,%u}",
             (int)r, (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2,
             (unsigned long long)stride1_bytes, (unsigned long long)stride2_bytes, box0, box1);
    set_error_text(msg);
    return NNAB_ECUDA;
  }
  return NNAB_OK;
}

// 4-D bf16 map, box {box0, box1, box2, 1}, swizzle by bk as encode_3d; strides in bytes for dims 1..3 (any order
// of magnitude: a dimension may step by less than the extent of the one below it -- overlapping views)
int encode_4d(CUtensorMap* map, void* base, const uint64_t dims[4], const uint64_t strides[3],
              const uint32_t box[3], int bk) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) {
    set_error_text("cuTensorMapEncodeTiled entry point not available");
    return NNAB_ECUDA;
  }
  cuuint64_t gdim[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t gstr[3] = {strides[0], strides[1], strides[2]};
  cuuint32_t bx[4] = {box[0], box[1], box[2], 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, base, gdim, gstr, bx, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE,
                        (bk == 64) ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[240];
    snprintf(msg, sizeof(msg),
             "cuTensorMapEncodeTiled(4d) failed (%d): dims {%llu,%llu,%llu,%llu} strides {%llu,%llu,%llu}",
             (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
             (unsigned long long)dims[3], (unsigned long long)strides[0], (unsigned long long)strides[1],
             (unsigned long long)strides[2]);
    set_error_text(msg);
    return NNAB_ECUDA;
  }
  return NNAB_OK;
}

int usable_sms(int* sms) {
  int dev = 0;
  NNAB_CUDA_TRY(cudaGetDevice(&dev));
  NNAB_CUDA_TRY(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
  *sms -= sm_reserve();
  if (*sms < 1) *sms = 1;
  return NNAB_OK;
}

EpiParams epilogue_of(const FramedProblem& q) {
  EpiParams e{};
  e.scale = q.scale; e.scale_all = q.scale_all; e.fmt = q.fmt;
  e.eps = q.eps; e.power = q.power; e.out = q.out; e.T = q.T;
  e.out_bins = q.out_bins; e.bin_offset = q.bin_offset; e.F = q.F;
  e.fb_table = q.fb_table; e.fb_steps = q.fb_steps; e.n_fb = q.n_fb;
  e.dec = q.dec;
  e.ola_pitch = q.ola_pitch; e.ola_hop = q.ola_hop;
  e.planes_stride = q.planes_stride; e.planes_pitch = q.planes_pitch;
  return e;
}

template <int FMT>
static int launch_tc_kernel_fmt(const CUtensorMap& ma, const CUtensorMap& mb, const TcParams& prm,
                                int grid, cudaStream_t stream) {
  return launch_persistent<framed_tc_kernel<FMT>>(grid, TC_KERNEL_THREADS, TcSmem::TOTAL, TcSmem::TOTAL, stream,
                                                  ma, mb, prm);
}

static int launch_tc_kernel(const CUtensorMap& ma, const CUtensorMap& mb, const TcParams& prm,
                            int grid, cudaStream_t stream) {
  switch (prm.epi.fmt) {
    case NNAB_FMT_MAGNITUDE: return launch_tc_kernel_fmt<0>(ma, mb, prm, grid, stream);
    case NNAB_FMT_COMPLEX: return launch_tc_kernel_fmt<1>(ma, mb, prm, grid, stream);
    case NNAB_FMT_PHASE_ANGLE: return launch_tc_kernel_fmt<2>(ma, mb, prm, grid, stream);
    case NNAB_FMT_PHASE_UNIT: return launch_tc_kernel_fmt<3>(ma, mb, prm, grid, stream);
    case FMT_POWER: return launch_tc_kernel_fmt<4>(ma, mb, prm, grid, stream);
    case FMT_FBANK: return launch_tc_kernel_fmt<5>(ma, mb, prm, grid, stream);
    case FMT_DECIM: return launch_tc_kernel_fmt<6>(ma, mb, prm, grid, stream);
    case FMT_RAW: return launch_tc_kernel_fmt<7>(ma, mb, prm, grid, stream);
    case FMT_OLA: return launch_tc_kernel_fmt<8>(ma, mb, prm, grid, stream);
    case FMT_REALPAIR: return launch_tc_kernel_fmt<9>(ma, mb, prm, grid, stream);
    default: return NNAB_EINVAL;
  }
}


// ---------------------------------------------------------------------------
// layout of a packed basis, keyed by its device pointer.  Every function that produces a buffer for the
// `packed` argument of launch_framed_tc sets (or clears) the entry, so a recycled address cannot carry a
// stale layout.
// ---------------------------------------------------------------------------
struct PackedLayout { int kind, n_fft, hop; };
static std::mutex g_pack_mu;
static std::unordered_map<const void*, PackedLayout> g_packed;

int packed_kind(const void* packed, int* n_fft, int* hop) {
  std::lock_guard<std::mutex> lk(g_pack_mu);
  auto it = g_packed.find(packed);
  const PackedLayout l = it == g_packed.end() ? PackedLayout{PACK_DENSE, 0, 0} : it->second;
  if (n_fft) *n_fft = l.n_fft;
  if (hop) *hop = l.hop;
  return l.kind;
}

void mark_packed(const void* packed, int kind, int n_fft, int hop) {
  std::lock_guard<std::mutex> lk(g_pack_mu);
  if (kind == PACK_DENSE) g_packed.erase(packed);
  else g_packed[packed] = PackedLayout{kind, n_fft, hop};
}


// ---------------------------------------------------------------------------
// per-K-block MMA width, host side (layout NNAB_LAYOUT_GROUPS)
// ---------------------------------------------------------------------------
bool tc_varn_basis_ok(int F, int K) { return F >= 1 && F <= 128 && K >= 64 && K <= 64 * VN_MAX_BLOCKS; }

int tc_pack_basis_varn(const float* w_re, const float* w_im, int F, int K, void* packed,
                       cudaStream_t stream) {
  if (!tc_varn_basis_ok(F, K)) return NNAB_EINVAL;
  const int rows = 16 * ((F + 7) / 8);
  const int kpad = round_up_i(K, 64);
  const int64_t threads = (int64_t)rows * (kpad / 8);
  pack_basis_varn_kernel<<<(unsigned)ceil_div64(threads, 256), 256, 0, stream>>>(
      w_re, w_im, F, K, rows, kpad, (__nv_bfloat16*)packed);
  NNAB_LAUNCH_CHECK();
  mark_packed(packed, PACK_VARN);
  return NNAB_OK;
}

// Pure host: which K blocks are touched, by how many 8-bin groups, in which order, and how the
// ordered list is cut into split-K chunks of equal modelled cost (max(N, 64) per block: below
// N = 64 the A-operand reads, not the MMA, set the pace).  Returns NNAB_OK or NNAB_EUNSUPPORTED.
int tc_varn_plan(const int32_t* k_begin, const int32_t* k_end, int F, int K, int want_chunks,
                 VarNPlan* plan) {
  const int nkb = (K + 63) / 64;
  if (nkb > VN_MAX_BLOCKS || F > 128 || F < 1) return NNAB_EUNSUPPORTED;
  std::vector<std::pair<int, int>> blocks;  // (groups, kb)
  for (int kb = 0; kb < nkb; ++kb) {
    int gmax = 0;
    for (int f = 0; f < F; ++f) {
      const int lo = k_begin ? k_begin[f] : 0, hi = k_end ? k_end[f] : K;
      if (hi > lo && hi > kb * 64 && lo < kb * 64 + 64) gmax = std::max(gmax, f / 8 + 1);
    }
    if (gmax > 0) blocks.push_back({gmax, kb});
  }
  if (blocks.empty()) blocks.push_back({(F + 7) / 8, 0});
  std::stable_sort(blocks.begin(), blocks.end(),
                   [](const std::pair<int, int>& a, const std::pair<int, int>& b) { return a.first > b.first; });
  plan->n_blocks = (int)blocks.size();
  int64_t total = 0;
  for (int i = 0; i < plan->n_blocks; ++i) {
    plan->groups[i] = (uint8_t)blocks[i].first;
    plan->order[i] = (uint16_t)blocks[i].second;
    total += std::max(16 * blocks[i].first, 64);
  }
  int chunks = want_chunks < 1 ? 1 : (want_chunks > 16 ? 16 : want_chunks);
  if (chunks > plan->n_blocks) chunks = plan->n_blocks;
  plan->n_chunks = chunks;
  plan->chunk_begin[0] = 0;
  int64_t acc = 0;
  int c = 1;
  for (int i = 0; i < plan->n_blocks && c < chunks; ++i) {
    acc += std::max(16 * (int)plan->groups[i], 64);
    // close chunk c-1 once its share of the cost is reached, leaving >= 1 block per later chunk
    if (acc * chunks >= total * c && plan->n_blocks - (i + 1) >= chunks - c) plan->chunk_begin[c++] = i + 1;
  }
  while (c < chunks) { plan->chunk_begin[c] = plan->n_blocks - (chunks - c); ++c; }
  plan->chunk_begin[chunks] = plan->n_blocks;
  for (int k = chunks + 1; k < 17; ++k) plan->chunk_begin[k] = plan->n_blocks;
  return NNAB_OK;
}

// host-only view of the plan for tests / tooling
int tc_varn_plan_export(const int32_t* k_begin, const int32_t* k_end, int F, int K, int want_chunks,
                        int32_t* order, int32_t* groups, int32_t* chunk_begin, int32_t* n_blocks,
                        int32_t* n_chunks) {
  VarNPlan plan;
  const int rc = tc_varn_plan(k_begin, k_end, F, K, want_chunks, &plan);
  if (rc) return rc;
  *n_blocks = plan.n_blocks;
  *n_chunks = plan.n_chunks;
  for (int i = 0; i < plan.n_blocks; ++i) { order[i] = plan.order[i]; groups[i] = plan.groups[i]; }
  for (int c = 0; c <= plan.n_chunks; ++c) chunk_begin[c] = plan.chunk_begin[c];
  return NNAB_OK;
}

static bool varn_problem_ok(const FramedProblem& q) {
  if (!tc_varn_basis_ok(q.F, q.K)) return false;
  if (num_phases(q.hop) != 1 || q.presplit != nullptr) return false;
  if (q.bin_offset != 0 || q.out_bins != q.F) return false;
  return q.fmt == NNAB_FMT_MAGNITUDE || q.fmt == NNAB_FMT_COMPLEX || q.fmt == NNAB_FMT_PHASE_UNIT;
}

template <int FMT>
static int launch_tcv_fmt(const CUtensorMap& ma, const CUtensorMap& mb8, const CUtensorMap& mb32,
                          const TcParams& prm, const VarNPlan& plan, int grid, cudaStream_t stream) {
  return launch_persistent<framed_tcv_kernel<FMT>>(grid, TC_KERNEL_THREADS, TcSmem::TOTAL, TcSmem::TOTAL, stream,
                                                   ma, mb8, mb32, prm, plan);
}

// The front half of the dense and VarN launchers: q's split-signal planes (the caller's pre-split planes, or the
// workspace with its K-overhang tail zeroed), their A-operand map and the SMs of the launch.  split_phase then
// writes the planes of each frame phase.
struct FramedSignal {
  SplitGeom g;
  int n_ph, hop_eff;
  int rows_mode;  // 1: A viewed as a (rows x hop_eff) matrix (64 | hop_eff); 0: overlapping-stride map
  __nv_bfloat16* planes;
  int sms;
  CUtensorMap ma;
};

static int framed_signal(const FramedProblem& q, void* workspace, size_t ws_bytes, cudaStream_t stream,
                         FramedSignal* s) {
  if (q.presplit == nullptr) {
    const size_t need = tc_workspace_bytes(q.B, q.L, q.K, q.hop, q.pad);
    if (workspace == nullptr || ws_bytes < need) return NNAB_EWORKSPACE;
  } else if (num_phases(q.hop) != 1) {
    return NNAB_EALIGN;  // pre-split planes exist for one frame phase only
  }
  if (q.B > 65535) return NNAB_EUNSUPPORTED;
  s->n_ph = num_phases(q.hop);
  s->hop_eff = q.hop * s->n_ph;
  SplitGeom& g = s->g;
  g = split_geom(q.B, q.L, q.K, q.hop, q.pad);
  if (q.presplit != nullptr && q.presplit_t_slots > 0) {
    // caller-defined plane geometry (pyramid levels shared with the FIR stage): frame g of the batch
    // still starts at element g * hop, with presplit_t_slots frames per clip slot
    g.t_slots = q.presplit_t_slots;
    g.nv = q.B * g.t_slots;
    g.plane_stride = q.presplit_plane_stride;
    g.rows = g.plane_stride / s->hop_eff;
    if (g.rows < g.nv) return NNAB_EINVAL;
  }
  int rc;
  if (q.presplit != nullptr) {
    s->planes = reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(q.presplit));
  } else {
    s->planes = reinterpret_cast<__nv_bfloat16*>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    if ((rc = zero_tail(s->planes, g.nv * s->hop_eff, g.plane_stride, stream))) return rc;
  }
  if ((rc = usable_sms(&s->sms))) return rc;
  s->rows_mode = (s->hop_eff % 64 == 0) ? 1 : 0;
  if (s->rows_mode)
    return encode_3d(&s->ma, s->planes, (uint64_t)s->hop_eff, (uint64_t)g.rows, 2, (uint64_t)s->hop_eff * 2,
                     (uint64_t)g.plane_stride * 2, 64, TC_BM, 64);
  // overlapping rows: row g starts at element g * hop_eff and is kpad long
  return encode_3d(&s->ma, s->planes, (uint64_t)round_up_i(q.K, 64), (uint64_t)g.nv, 2, (uint64_t)s->hop_eff * 2,
                   (uint64_t)g.plane_stride * 2, 64, TC_BM, 64);
}

// the planes of frame phase ph: the signal shifted by ph * hop samples (pre-split planes are the caller's)
static int split_phase(const FramedProblem& q, const FramedSignal& s, int ph, cudaStream_t stream) {
  if (q.presplit != nullptr) return NNAB_OK;
  const int64_t clip_pitch = s.g.t_slots * s.hop_eff;
  dim3 grid((unsigned)ceil_div64(clip_pitch, 256 * 8), (unsigned)q.B);
  return launch_problem_split(q, grid, ph * q.hop, clip_pitch, s.g.plane_stride, 0, s.planes, stream);
}

// Split-K (long kernels, with the caller's raw scratch): the kernel writes raw (re, im) partial sums to the
// scratch, and splitk_finalize_kernel then applies the returned epilogue to them.
static EpiParams use_splitk_scratch(const FramedProblem& q, EpiParams* e) {
  e->raw = reinterpret_cast<float*>(((uintptr_t)q.raw + 255) & ~(uintptr_t)255);
  e->raw_plane = (int64_t)q.B * q.F * q.T;
  const EpiParams final_epi = *e;
  e->fmt = FMT_RAW;
  return final_epi;
}

static int launch_splitk_finalize(const EpiParams& e, int64_t B, cudaStream_t stream) {
  dim3 grid((unsigned)ceil_div64(e.T, 256), (unsigned)e.F, (unsigned)(B < 64 ? B : 64));
  splitk_finalize_kernel<<<grid, 256, 0, stream>>>(e, B);
  NNAB_LAUNCH_CHECK();
  return NNAB_OK;
}

static int launch_framed_tc_varn(const FramedProblem& q, const void* packed, void* workspace,
                                 size_t ws_bytes, cudaStream_t stream) {
  if (!varn_problem_ok(q)) return NNAB_EINVAL;  // the basis was packed for this kernel only
  {
    // same packed layout, A operand read in place from one tall block per column (tct_kernels.cu)
    const int trc = launch_framed_tc_tall(q, packed, workspace, ws_bytes, stream);
    if (trc != NNAB_EUNSUPPORTED) return trc;
  }
  FramedSignal s;
  int rc = framed_signal(q, workspace, ws_bytes, stream, &s);
  if (rc) return rc;
  if ((rc = split_phase(q, s, 0, stream))) return rc;  // one frame phase (varn_problem_ok)
  const int kpad = round_up_i(q.K, 64);
  const int rows_w = 16 * ((q.F + 7) / 8);

  // split-K only with the caller's raw scratch (long kernels): <= 64 K blocks per accumulator
  VarNPlan plan;
  {
    VarNPlan probe;
    if ((rc = tc_varn_plan(q.h_k_begin, q.h_k_end, q.F, q.K, 1, &probe))) return rc;
    int ks = 1;
    if (q.raw != nullptr) {
      ks = (probe.n_blocks + 63) / 64;
      if (ks > 16) ks = 16;
    }
    if ((rc = tc_varn_plan(q.h_k_begin, q.h_k_end, q.F, q.K, ks, &plan))) return rc;
  }

  CUtensorMap mb8, mb32;
  if ((rc = encode_3d(&mb8, const_cast<void*>(packed), (uint64_t)kpad, (uint64_t)rows_w, 2,
                      (uint64_t)kpad * 2, (uint64_t)rows_w * kpad * 2, 64, 8, 64)))
    return rc;
  if ((rc = encode_3d(&mb32, const_cast<void*>(packed), (uint64_t)kpad, (uint64_t)rows_w, 2,
                      (uint64_t)kpad * 2, (uint64_t)rows_w * kpad * 2, 64, 32, 64)))
    return rc;

  TcParams prm{};
  prm.num_n_tiles = 1;
  prm.bn = rows_w;
  prm.rows_mode = s.rows_mode;
  prm.hop = s.hop_eff;
  prm.nv = s.g.nv;
  prm.t_slots = s.g.t_slots;
  prm.t_mul = 1;
  prm.t_add = 0;
  prm.T = q.T;
  prm.k_splits = plan.n_chunks;
  prm.epi = epilogue_of(q);
  prm.epi.fb_table = nullptr;
  const bool split = plan.n_chunks > 1;
  const EpiParams final_epi = split ? use_splitk_scratch(q, &prm.epi) : prm.epi;
  prm.num_m_tiles = (int)ceil_div64(s.g.nv, TC_BM);
  const int64_t units = (int64_t)prm.num_m_tiles * plan.n_chunks;
  const int grid = (int)(units < s.sms ? units : s.sms);
  {
    double cols = 0.0;
    for (int i = 0; i < plan.n_blocks; ++i) cols += 16.0 * plan.groups[i] * 64.0;
    add_exec_flops(3.0 * 2.0 * (double)prm.num_m_tiles * TC_BM * cols);
  }
  switch (prm.epi.fmt) {
    case NNAB_FMT_MAGNITUDE: rc = launch_tcv_fmt<0>(s.ma, mb8, mb32, prm, plan, grid, stream); break;
    case NNAB_FMT_COMPLEX: rc = launch_tcv_fmt<1>(s.ma, mb8, mb32, prm, plan, grid, stream); break;
    case NNAB_FMT_PHASE_UNIT: rc = launch_tcv_fmt<3>(s.ma, mb8, mb32, prm, plan, grid, stream); break;
    case FMT_RAW: rc = launch_tcv_fmt<7>(s.ma, mb8, mb32, prm, plan, grid, stream); break;
    default: rc = NNAB_EINVAL;
  }
  if (rc) return rc;
  if (split && (rc = launch_splitk_finalize(final_epi, q.B, stream))) return rc;
  if (q.route != nullptr) *q.route = split ? NNAB_CQ1992_VARN_SPLITK : NNAB_CQ1992_VARN;
  return NNAB_OK;
}

int launch_framed_tc(const FramedProblem& q, const void* packed, void* workspace, size_t ws_bytes,
                     cudaStream_t stream) {
  if (q.B <= 0 || q.T <= 0 || q.F <= 0) return NNAB_OK;
  if (packed == nullptr) return NNAB_EINVAL;
  const int kind = packed_kind(packed);
  if (kind == PACK_BLOCK) return launch_framed_tc_block(q, packed, workspace, ws_bytes, stream);
  if (kind == PACK_VARN) return launch_framed_tc_varn(q, packed, workspace, ws_bytes, stream);
  FramedSignal s;
  int rc = framed_signal(q, workspace, ws_bytes, stream, &s);
  if (rc) return rc;

  constexpr int bk = 64;
  const int n_ph = s.n_ph;
  const int kpad = round_up_i(q.K, 64);
  // FMT_OLA: the N axis is the frame's n_fft output samples (q.F), not (re | im) bin pairs
  OlaPlan ola{};
  if (q.fmt == FMT_OLA) {
    ola = tc_ola_plan(q.F, q.K, s.g.nv, q.k_splits_hint);
    if (!ola.supported || q.h_k_begin != nullptr) return NNAB_EINVAL;
  }
  const int bn = (q.fmt == FMT_OLA) ? ola.bn : choose_bn(q.F);
  const int n_tiles = (q.fmt == FMT_OLA) ? ola.n_tiles : (2 * q.F + bn - 1) / bn;
  const int rows_w = n_tiles * bn;
  CUtensorMap mb;
  rc = encode_3d(&mb, const_cast<void*>(packed), (uint64_t)kpad, (uint64_t)rows_w, 2,
                 (uint64_t)kpad * 2, (uint64_t)rows_w * kpad * 2, bk, bn, bk);
  if (rc) return rc;

  // ---- parameters -------------------------------------------------------------------
  TcParams prm{};
  prm.num_n_tiles = n_tiles;
  prm.bn = bn;
  prm.rows_mode = s.rows_mode;
  prm.hop = s.hop_eff;
  prm.nv = s.g.nv;
  prm.t_slots = s.g.t_slots;
  prm.t_mul = n_ph;
  const int nkb = kpad / bk;
  const int half = bn / 2;
  for (int tl = 0; tl < n_tiles; ++tl) {
    int lo = 0, hi = (q.K + bk - 1) / bk;
    if (q.h_k_begin != nullptr && q.h_k_end != nullptr) {
      int klo = q.K, khi = 0;
      for (int f = tl * half; f < q.F && f < (tl + 1) * half; ++f)
        if (q.h_k_end[f] > q.h_k_begin[f]) {
          klo = q.h_k_begin[f] < klo ? q.h_k_begin[f] : klo;
          khi = q.h_k_end[f] > khi ? q.h_k_end[f] : khi;
        }
      if (khi > klo) {
        lo = klo / bk;
        hi = (khi + bk - 1) / bk;
      } else {
        lo = 0;
        hi = 1;
      }
    }
    if (hi > nkb) hi = nkb;
    if (lo >= hi) lo = hi - 1;
    prm.kb_begin[tl] = lo;
    prm.kb_end[tl] = hi;
  }
  prm.epi = epilogue_of(q);
  prm.k_splits = 1;
  if (q.fmt == FMT_FBANK && (q.fb_table == nullptr || q.n_fb <= 0)) return NNAB_EINVAL;
  if (q.fmt == FMT_DECIM && (bn != 128 || n_tiles != 1)) return NNAB_EINVAL;

  if (q.fmt == FMT_OLA) prm.k_splits = ola.k_splits;  // the OLA atomics accumulate K chunks as is

  // ---- split-K (long kernels, caller supplied the raw scratch) ---------------------------
  EpiParams final_epi = prm.epi;
  bool split = false;
  if (q.raw != nullptr && q.fmt != FMT_FBANK && q.fmt != FMT_DECIM && q.fmt != FMT_OLA &&
      q.bin_offset == 0 &&
      q.out_bins == q.F) {
    int min_range = nkb;
    for (int tl = 0; tl < n_tiles; ++tl) {
      const int r = prm.kb_end[tl] - prm.kb_begin[tl];
      min_range = r < min_range ? r : min_range;
    }
    int ks = (min_range + 63) / 64;  // <= 64 k-blocks (4096 taps) per accumulator
    if (ks > 16) ks = 16;
    if (ks > min_range) ks = min_range;
    if (ks > 1) {
      split = true;
      prm.k_splits = ks;
      final_epi = use_splitk_scratch(q, &prm.epi);
    }
  }

  // ---- one pad/split + GEMM pass per frame phase ----------------------------------------
  for (int ph = 0; ph < n_ph; ++ph) {
    if (ph >= q.T) break;
    prm.t_add = ph;
    prm.T = (q.T - ph + n_ph - 1) / n_ph;  // frames t = ph, ph + n_ph, ... < T
    if ((rc = split_phase(q, s, ph, stream))) return rc;
    {
      double kcols = 0.0;  // sum over N tiles of (k-blocks executed) x bk x bn
      for (int tl = 0; tl < n_tiles; ++tl) kcols += (double)(prm.kb_end[tl] - prm.kb_begin[tl]) * bk * bn;
      add_exec_flops(3.0 * 2.0 * (double)ceil_div64(s.g.nv, TC_BM) * TC_BM * kcols);
    }
    prm.num_m_tiles = (int)ceil_div64(s.g.nv, TC_BM);
    const int64_t tiles = (int64_t)prm.num_m_tiles * prm.num_n_tiles * prm.k_splits;
    const int grid = (int)(tiles < s.sms ? tiles : s.sms);
    rc = launch_tc_kernel(s.ma, mb, prm, grid, stream);
    if (rc) return rc;
  }
  if (split && (rc = launch_splitk_finalize(final_epi, q.B, stream))) return rc;
  if (q.route != nullptr) *q.route = split ? NNAB_CQ1992_DENSE_SPLITK : NNAB_CQ1992_DENSE;
  return NNAB_OK;
}

}  // namespace nnab
