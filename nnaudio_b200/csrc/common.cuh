// Shared declarations for libnnab.so (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "nnab.h"

namespace nnab {

// ---- error plumbing -------------------------------------------------------
void set_cuda_error(const char* where, cudaError_t e);
void set_error_text(const char* text);
void count_launch();
void count_balanced_launch();
void count_block_ws_launch();
int sm_reserve();
// the persistent-grid ledger (nnab_persistent_grid_read): one persistent launch of `grid` CTAs
void count_persistent_grid(int grid);
// tensor-pipe accounting for bench.py: MMA flops a tensor-core launch EXECUTES (all split terms,
// tile padding and structural zeros included); summed while nnab_profile_enable(1)
void add_exec_flops(double flops);

#define NNAB_CUDA_TRY(expr)                         \
  do {                                              \
    cudaError_t _e = (expr);                        \
    if (_e != cudaSuccess) {                        \
      ::nnab::set_cuda_error(#expr, _e);            \
      return NNAB_ECUDA;                            \
    }                                               \
  } while (0)

#define NNAB_LAUNCH_CHECK()                         \
  do {                                              \
    ::nnab::count_launch();                         \
    cudaError_t _e = cudaGetLastError();            \
    if (_e != cudaSuccess) {                        \
      ::nnab::set_cuda_error("kernel launch", _e);  \
      return NNAB_ECUDA;                            \
    }                                               \
  } while (0)

// ---- problem description shared by the SIMT and tensor-core framed kernels ----
// One "framed complex contraction":
//   re[b,f,t] = sum_k xpad[b, t*hop + k] * w_re[f,k]
//   im[b,f,t] = -sum_k xpad[b, t*hop + k] * w_im[f,k]
// followed by a per-bin scale and one of the output formats of nnab.h (or the
// internal POWER format used by the filterbank ops).
constexpr int FMT_POWER = 100;  // internal: (sqrt(re^2+im^2+eps)) ** power -> (B,F,T)
constexpr int FMT_FBANK = 101;  // internal (tensor-core only): power -> banded filterbank -> (B,n_fb,T)
constexpr int FMT_DECIM = 102;  // internal (tensor-core only): FIR decimator stage of the CQT pyramid
constexpr int FMT_RAW = 103;    // internal (tensor-core only): split-K partial sums -> raw (re, im) scratch
constexpr int FMT_OLA = 104;    // internal (tensor-core only): inverse STFT frames -> overlap-add buffer
constexpr int FMT_PLANES = 105;   // internal (block-partial kernel only): power spectrum -> bf16 hi/lo operand
                                  //   planes of the dense-filterbank GEMM (`out` = plane base, see planes_*)
constexpr int FMT_REALPAIR = 106; // internal (dense tensor-core kernel only): two real outputs per complex column
                                  //   pair: re -> row f, im -> row f + F of a real (B, out_bins, T) tensor

// FMT_DECIM epilogue target: the NEXT pyramid level, written as bf16 hi/lo planes in
// the layout the tensor-core kernels read (sample m of clip b at b*pitch + off + m).
//   pc: input of the level's octave CQT — reflect (or zero) margins of `pc_off` samples
//   pf: input of the level's own FIR stage — zero margins, samples at offset 128
//   y32: optional fp32 copy (levels whose hop needs several frame phases)
struct DecimParams {
  void* pc; int64_t pc_plane, pc_pitch; int pc_off, pc_reflect;
  void* pf; int64_t pf_plane, pf_pitch;
  float* y32; int64_t y32_pitch;
  int64_t len_out;  // valid samples per clip of the next level
};

// Banded filterbank table: the (at most two) non-zero weights of every FFT bin.
struct FbEntry {
  int j0, j1;    // filter rows (-1 = none)
  float w0, w1;
};

// Static action list of the banded-filterbank epilogue (block-partial kernel): what the two running
// filter sums of a row do at FFT bin k -- the control flow depends on k only, so it is resolved once
// per filterbank instead of per (row, bin).  Before accumulating bin k: a slot whose flush id is
// >= 0 adds its sum to that filter's output and restarts from zero; then slot a += wa * P[k],
// slot b += wb * P[k].  cur_a / cur_b = filters the slots hold after bin k (flushed at a range end).
struct FbStep {
  float wa, wb;
  short flush_a, flush_b;
  short cur_a, cur_b;
};
static_assert(sizeof(FbStep) == 16, "one 128-bit load per bin");
constexpr int FB_STEP_PAD = 160;  // entries past F (a tile's last chunk may overrun the last bin)
// epilogue warps per 32-row quarter of the fused-filterbank block kernel: each covers a contiguous
// range of a tile's 8-column chunks, [n_chunks * part / PARTS, n_chunks * (part + 1) / PARTS)
// (with 3, a 53-bin mel filter spans three ranges, its three atomic partial sums no longer commute and
// results differ run to run: 2 it is.)
constexpr int FB_EPI_PARTS = 2;

// The four-phase block kernel (tcb_kernels.cu) emits bin k of an n_fft = 4 M transform (F = 2 M + 1) from one
// of four "families" of the M-point phase DFTs, each over k' = 0 .. M/2:
//   f0 [0, M/2): k' = k    f1 [M/2, M): k' = M - k    f2 [M, 3M/2): k' = k - M    f3 [3M/2, 2M]: k' = 2M - k
// Tile t of width nb holds k' in [t (nb - 2), (t + 1)(nb - 2)); f1 and f3 run reversed inside it, so that every
// family emits ascending bins: output position o = k' - t (nb - 2) for f0 / f2, nb - 3 - that for f1 / f3.
// The two warps of a family quarter (column parts) hand the sums of the filters open at their cut over inside
// the CTA, so the range that adds one partial sum to each filter it meets (fused filterbank) is (family, tile).
__host__ __device__ inline int poly4_family(int k, int M, int* kq) {
  const int f = k < M / 2 ? 0 : (k < M ? 1 : (k < 3 * M / 2 ? 2 : 3));
  *kq = (f == 0) ? k : (f == 1 ? M - k : (f == 2 ? k - M : 2 * M - k));
  return f;
}
// Bins of family f in tile n: output o (0 <= o < nb - 2) is bin *k0 + o, and the family emits it iff it lies in
// [*lo, *hi).  M = 0 is the one-phase kernel: one family, bins n (nb - 2) + o below F.
__host__ __device__ inline void block_family_span(int n, int f, int nb, int M, int F, int* k0, int* lo, int* hi) {
  const int kq0 = n * (nb - 2);
  if (M == 0) {
    *k0 = kq0; *lo = 0; *hi = F;
    return;
  }
  *k0 = (f == 0) ? kq0 : (f == 1 ? M - kq0 - (nb - 3) : (f == 2 ? M + kq0 : 2 * M - kq0 - (nb - 3)));
  *lo = f * (M / 2);
  const int h = (f == 3) ? 2 * M + 1 : (f + 1) * (M / 2);
  *hi = h < F ? h : F;
}
__host__ __device__ inline int poly4_range(int k, int M, int nb) {
  int kq;
  const int f = poly4_family(k, M, &kq);
  return f * 4096 + kq / (nb - 2);
}

// The signals of one push of chunked streams (DESIGN §3.10): batch row b is the "virtual clip" of `length`
// samples of one stream, lane b of the push.  The lane names the stream's ring row and chunk row (`slot`), its
// counters and its end; the clip's sample i is the stream's raw sample r = frames * hop - pad + i.  Raw samples
// [.., received) come from the fp32 carry ring (raw r of slot s at ring[s * ring_pitch + r % ring_len]),
// [received, received + n) from the chunk (samples of type FramedProblem::x_dtype, rows of chunk_pitch).
// r < 0 is the left centre padding; on the stream's last push (end) r >= received + n is the right one.  The
// clip length is the batch's longest; a row's samples past its own stream read as zeros.
// Lane b is lanes[b] of the DEVICE lane table (stream pools), or without one (a lock-step push of B streams
// that share one set of counters) `shared` in slot b.
struct PyrLaneSig;
struct ChunkSource {
  const float* ring;
  int64_t ring_pitch;
  int64_t ring_len;
  const void* chunk;
  int64_t chunk_pitch;
  int64_t length;
  int pad_mode;
  const nnab_stream_lane* lanes;
  nnab_stream_lane shared;        // lane b when lanes == nullptr (slot = b)
  int K, hop, pad;                // the framing that places each lane's clip
  // pyramid pools (rows != nullptr, lanes == nullptr): row b of the launch takes everything from the DEVICE
  // descriptor rows[b] (PyrLaneSig below): its ring row, its source row and base, its counts, and -- rows_oct = 1,
  // an octave clip (pad: the octave's) -- the octave's frame origin, padding and end, or -- rows_oct = 0, a FIR
  // stage source -- the stage's source origin, with zeros past the row's samples.
  const PyrLaneSig* rows;
  int rows_oct;
};

// ---- the counters of one stream (DESIGN §3.10), shared by the host checks and the pool kernels ----------
// Frame t is returned by the first push after which every raw sample it reads has arrived: t * hop + K - pad
// samples (reflect padding: and at least pad + 1, the left mirror of frame 0), or all remaining frames on
// the last push.
__host__ __device__ inline int64_t chunk_ready_frames(int64_t total, int K, int hop, int pad, int pad_mode) {
  if (pad > 0 && pad_mode == NNAB_PAD_REFLECT && total < pad + 1) return 0;
  const int64_t need = (int64_t)K - pad;
  return total < need ? 0 : (total - need) / hop + 1;
}

// Frames of the whole stream of `total` samples, once it has ended (the offline call's T).
__host__ __device__ inline int64_t chunk_end_frames(int64_t total, int K, int hop, int pad) {
  const int64_t span = total + 2 * (int64_t)pad - K;
  return span < 0 ? 0 : span / hop + 1;
}

// First raw sample the push after `frames` frames still reads: the first frame's start, and with centre
// padding no later than total - (pad + 1) (the right mirror of the last push reads that far back).
__host__ __device__ inline int64_t chunk_carry_start(int64_t total, int64_t frames, int hop, int pad) {
  int64_t s = frames * hop - pad;
  if (pad > 0 && s > total - (pad + 1)) s = total - (pad + 1);
  if (s < 0) s = 0;
  return s < total ? s : total;
}

// Host counters of a stream: `received` raw samples so far, the last `n_carry` of them in the carry ring,
// `frames` frames returned.
struct StreamStep {
  int64_t total;      // raw samples after the push
  int64_t t_end;      // frames returned after the push
  int64_t T;          // frames this push returns
  int64_t from;       // raw samples [from, total) go into the ring after the push
};

// One push of one stream: n new samples, the last push iff `end`.  NNAB_EINVAL for counters no stream can
// have (they must be those of a stream that returned every ready frame) and for an end the stream is too
// short for (reflect padding needs pad < total; at least one frame).  Every lane of a push is checked here: the
// one lane the B streams of *_chunk_forward share, each lane of a pool's table and every slot of a device pool's
// plan launch.
__host__ __device__ inline int stream_step(int64_t received, int64_t n_carry, int64_t frames, int64_t n, int end,
                                           int K, int hop, int pad, int pad_mode, StreamStep* o) {
  if (received < 0 || frames < 0 || n < 0) return NNAB_EINVAL;
  if (frames != chunk_ready_frames(received, K, hop, pad, pad_mode) ||
      n_carry != received - chunk_carry_start(received, frames, hop, pad))
    return NNAB_EINVAL;
  const int64_t total = received + n;
  int64_t t_end;
  if (end) {
    if (pad > 0 && pad_mode == NNAB_PAD_REFLECT && pad >= total) return NNAB_EINVAL;
    t_end = chunk_end_frames(total, K, hop, pad);
    if (t_end <= 0) return NNAB_EINVAL;
  } else {
    t_end = chunk_ready_frames(total, K, hop, pad, pad_mode);
  }
  o->total = total;
  o->t_end = t_end;
  o->T = t_end - frames;
  const int64_t keep = chunk_carry_start(total, t_end, hop, pad);
  o->from = keep > received ? keep : received;
  return NNAB_OK;
}

// Frames a pool lane has returned after its push (the library has checked the lane on the host).
__host__ __device__ inline int64_t lane_frames_after(const nnab_stream_lane& ln, int K, int hop, int pad,
                                                     int pad_mode) {
  const int64_t total = ln.received + ln.n;
  return ln.end ? chunk_end_frames(total, K, hop, pad) : chunk_ready_frames(total, K, hop, pad, pad_mode);
}

// ---- the streamed CQT pyramid (DESIGN §3.10 "Pyramid streams"), shared by the host checks and the pool kernels
// Level lengths follow conv1d(stride=n, padding=127, kernel=256): (len - 2)/n + 1.
__host__ __device__ inline int64_t decimated_len(int64_t len, int factor) {
  return len < 2 ? 0 : (len - 2) / factor + 1;
}

// Signals of a stream: the raw samples when an early stage feeds level 0, then one per octave (octave i on
// signal i + e).  Stage s turns signal s into s + 1 (factor d[s]): y[n] = sum_m fir[m] x[d n + m - 127].
// Every per-signal number is a function of the raw count alone: before the end, sample n of signal s + 1 is
// final once d n + c of signal s have arrived -- c = 129 (its last tap reads d n + 128), 130 on the gen-2 plan,
// whose edge fix recomputes the last 64 outputs of the whole clip on the CUDA cores: with one sample more, n is
// never one of them.  Signal s keeps an fp32 ring (stream b at ring[b * len + r % len]) of what later pushes read.
struct PyrStream {
  int n_sig, e, n_oct, c;
  bool gen2;
  int d[33];
  int width[32], hop[32], pad[32];
  int64_t ring_len[33];
  size_t ring_off[33];  // floats
  size_t state_floats;  // per stream
};

// Samples of every signal after `raw` raw samples: final ones before the end, all of them on flush.
__host__ __device__ inline void pyr_counts(const PyrStream& p, int64_t raw, int flush, int64_t* R) {
  R[0] = raw;
  for (int s = 0; s + 1 < p.n_sig; ++s) {
    if (flush) R[s + 1] = decimated_len(R[s], p.d[s]);
    else R[s + 1] = R[s] >= p.c ? (R[s] - p.c) / p.d[s] + 1 : 0;
  }
}

// Frames final in every octave (before the end).
__host__ __device__ inline int64_t pyr_ready_frames(const PyrStream& p, const int64_t* R, int pad_mode) {
  int64_t t = INT64_MAX;
  for (int i = 0; i < p.n_oct; ++i) {
    const int64_t f = chunk_ready_frames(R[i + p.e], p.width[i], p.hop[i], p.pad[i], pad_mode);
    t = f < t ? f : t;
  }
  return t;
}

// First sample of signal s a later push reads, after `frames` frames with the counts R.
__host__ __device__ inline int64_t pyr_keep(const PyrStream& p, int s, const int64_t* R, int64_t frames) {
  int64_t k = R[s];
  const int l = s - p.e;
  if (l >= 0) k = chunk_carry_start(R[s], frames, p.hop[l], p.pad[l]);
  if (s + 1 < p.n_sig) {
    int64_t f = 128 * (int64_t)p.d[s] * (R[s + 1] / 128) - 128;
    f = f < 0 ? 0 : f;
    k = f < k ? f : k;
  }
  return k;
}

// The per-stream rules of one push (n new samples, the last push iff `end`): the counts before (R0) and after (R1)
// it, the frame bound after it and each octave's padding (reflect falls back to constant on a level the end leaves
// no longer than its pad).  NNAB_EINVAL for counters no stream can have (they must be those of a stream that
// returned every ready frame and carries what pyr_keep keeps), for an end the stream is too short for (a level
// left empty, an octave without frames, octave frame counts that differ, fewer frames than already returned) and
// for a push that would overrun a ring.  The one-stream push, every lane of a pool and every slot of a device
// pool's plan launch are checked here.
struct PyrStep {
  int64_t R0[33], R1[33];
  int64_t t_end;
  int mode[32];
};

__host__ __device__ inline int pyr_step(const PyrStream& p, int64_t received, int64_t n_carry, int64_t frames,
                                        int64_t n, int end, int pad_mode, PyrStep* o) {
  if (received < 0 || frames < 0 || n < 0) return NNAB_EINVAL;
  pyr_counts(p, received, 0, o->R0);
  if (frames != pyr_ready_frames(p, o->R0, pad_mode) || n_carry != received - pyr_keep(p, 0, o->R0, frames))
    return NNAB_EINVAL;
  pyr_counts(p, received + n, end, o->R1);
  for (int i = 0; i < p.n_oct; ++i) {
    const int64_t len = o->R1[i + p.e];
    o->mode[i] = (end && pad_mode == NNAB_PAD_REFLECT && p.pad[i] >= len) ? NNAB_PAD_CONSTANT : pad_mode;
  }
  if (end) {
    o->t_end = -1;
    for (int i = 0; i < p.n_oct; ++i) {
      const int64_t len = o->R1[i + p.e];
      if (len <= 0) return NNAB_EINVAL;
      const int64_t f = chunk_end_frames(len, p.width[i], p.hop[i], p.pad[i]);
      if (f <= 0 || (o->t_end >= 0 && f != o->t_end)) return NNAB_EINVAL;
      o->t_end = f;
    }
    if (o->t_end < frames) return NNAB_EINVAL;
  } else {
    o->t_end = pyr_ready_frames(p, o->R1, pad_mode);
    for (int s = 0; s < p.n_sig; ++s)
      if (o->R1[s] - pyr_keep(p, s, o->R1, o->t_end) > p.ring_len[s]) return NNAB_EINVAL;
  }
  return NNAB_OK;
}

// One pool lane's plan for signal s of a push: what the one-stream push (nnab_cqt_pyramid_chunk_forward) of the
// lane's counters does with that signal.  The plan kernel writes it per (signal, lane) into the workspace and
// every lane-aware kernel reads it; the host checks the lanes with the same functions first.
struct PyrLaneSig {
  int64_t slot;            // ring row
  int64_t R0, R1;          // final samples of the signal before and after the push
  int64_t keep;            // the ring keeps [keep, R1) after the push (R1 at an end: nothing)
  int64_t src_row, base;   // the new samples: source row (chunk row / new-sample row), sample R0 at `base`
  int64_t t0;              // first 128-output row of the FIR stage s -> s + 1 (-1: the lane has no new output)
  int64_t fir_origin;      // its source origin 128 d t0 - 128
  int64_t fir_len_src, fir_len_out;  // source samples / outputs from that row on (R1 - 128 d t0, R1' - 128 t0)
  int64_t oct_origin;      // the octave's first unreturned frame: frames * hop_l - pad_l
  int64_t count;           // frames the push returns (the lane's, the same on every signal)
  int32_t mode;            // the octave's padding (reflect falls back to constant on a short level at the end)
  int32_t end;
  int32_t head, tail;      // the FIR stage's CUDA-core edge fix: the stream's first / last 64 outputs
};

__host__ __device__ inline PyrLaneSig pyr_lane_signal(const PyrStream& p, const nnab_stream_lane& ln, int64_t lane,
                                                      int s, int pad_mode) {
  int64_t R0[33], R1[33];
  pyr_counts(p, ln.received, 0, R0);
  pyr_counts(p, ln.received + ln.n, (int)ln.end, R1);
  const int64_t t_end = ln.end ? chunk_end_frames(R1[p.e], p.width[0], p.hop[0], p.pad[0])
                               : pyr_ready_frames(p, R1, pad_mode);
  PyrLaneSig o{};
  o.slot = ln.slot;
  o.R0 = R0[s];
  o.R1 = R1[s];
  const int64_t k = ln.end ? R1[s] : pyr_keep(p, s, R1, t_end);
  o.keep = k > R0[s] ? k : R0[s];
  // the raw signal comes from the lane's chunk row; a decimated one from row `lane` of its new-sample buffer,
  // which holds the stage's outputs from its first row, 128 floor(R0 / 128), on
  o.src_row = s == 0 ? ln.slot : lane;
  o.base = s == 0 ? 0 : R0[s] % 128;
  o.t0 = -1;
  if (s + 1 < p.n_sig && R1[s + 1] > R0[s + 1]) {
    const int64_t t0 = R0[s + 1] / 128, d = p.d[s];
    o.t0 = t0;
    o.fir_origin = 128 * d * t0 - 128;
    o.fir_len_src = R1[s] - 128 * d * t0;
    o.fir_len_out = R1[s + 1] - 128 * t0;
    o.head = p.gen2 && t0 == 0;
    o.tail = p.gen2 && ln.end;
  }
  const int l = s - p.e;
  o.mode = pad_mode;
  if (l >= 0) {
    o.oct_origin = ln.frames * p.hop[l] - p.pad[l];
    if (ln.end && pad_mode == NNAB_PAD_REFLECT && p.pad[l] >= R1[s]) o.mode = NNAB_PAD_CONSTANT;
  }
  o.count = t_end - ln.frames;
  o.end = (int32_t)ln.end;
  return o;
}

// ---- the counters of one streamed inverse STFT (DESIGN §3.10), shared by the host checks and the pool kernels
// Overlap-add positions s (pad-cropped output sample s - offset).  After n frames, positions below n * hop are
// final; the output can still end as early as istft_end_min(n) (length None).
__host__ __device__ inline int64_t istft_end_min(int64_t n, int n_fft, int hop, int center) {
  const int64_t ola_len = n_fft + (int64_t)hop * (n - 1);
  return center ? ola_len - n_fft / 2 : ola_len;
}

struct IstftChunkPlan {
  int64_t origin;      // first position the push's overlap-add buffer holds (= first carried position)
  int64_t carried;     // positions carried in: [origin, origin + carried)
  int64_t buf_len;     // positions the push's buffer holds
  int64_t emit_begin, emit_end;
  int64_t carry_begin, carry_len;  // carried out
};

// Host counters: `frames` frames pushed so far, `emitted` output samples returned.  EINVAL for counters no
// stream has, or a `length` shorter than what was returned.
__host__ __device__ inline int istft_chunk_plan(int64_t frames, int64_t emitted, int64_t T, int n_fft, int hop,
                                                int center, int flush, int64_t length, IstftChunkPlan* o) {
  if (frames < 0 || emitted < 0 || T < 0 || n_fft <= 0 || hop <= 0 || hop > n_fft) return NNAB_EINVAL;
  const int64_t offset = center ? n_fft / 2 : 0;
  auto emitted_end = [&](int64_t n) {  // end of the positions returned by the pushes of n frames
    if (n <= 0) return offset;
    const int64_t e = n * hop < istft_end_min(n, n_fft, hop, center) ? n * hop : istft_end_min(n, n_fft, hop, center);
    return e > offset ? e : offset;
  };
  const int64_t E = emitted_end(frames);
  if (offset + emitted != E) return NNAB_EINVAL;
  const int64_t n = frames + T;
  if (flush && n <= 0) return NNAB_EINVAL;
  o->origin = frames > 0 ? (E < frames * hop ? E : frames * hop) : 0;
  o->carried = frames > 0 ? (frames - 1) * (int64_t)hop + n_fft - o->origin : 0;
  o->buf_len = n > 0 ? (n - 1) * (int64_t)hop + n_fft - o->origin : 0;
  o->emit_begin = E;
  if (flush) {
    const int64_t ola_len = n_fft + (int64_t)hop * (n - 1);
    int64_t want = length >= 0 ? length : (center ? ola_len - 2 * offset : ola_len);
    if (offset + want > ola_len) want = ola_len - offset;  // slicing past the end just truncates
    if (want < 0) want = 0;
    if (offset + want < E) return NNAB_EINVAL;  // shorter than the samples already returned
    o->emit_end = offset + want;
    o->carry_begin = o->carry_len = 0;
  } else {
    o->emit_end = emitted_end(n);
    const int64_t c = n > 0 ? (o->emit_end < n * hop ? o->emit_end : n * hop) : 0;
    o->carry_begin = c;
    o->carry_len = n > 0 ? (n - 1) * (int64_t)hop + n_fft - c : 0;
  }
  if (o->carried > n_fft || o->carry_len > n_fft) return NNAB_EINVAL;
  return NNAB_OK;
}

// A lane's plan on the device (the library has checked the lane on the host with the same function).
__host__ __device__ inline IstftChunkPlan istft_lane_plan(const nnab_istft_lane& ln, int n_fft, int hop,
                                                          int center) {
  IstftChunkPlan pl{};
  istft_chunk_plan(ln.frames, ln.emitted, ln.T, n_fft, hop, center, (int)ln.end, ln.end ? ln.length : -1, &pl);
  return pl;
}

// ---- device pools (DESIGN §3.10 "Device pools"): one slot's share of the plan launch, shared by the kernel and
// the host-only debug entry point.  counters is (3, slots); a dropped push leaves them as they are, writes an
// all-zero lane (no frame, no sample, no carry: the lane-aware kernels map it to nothing) and keeps the slot's
// first error code until its reset.
__host__ __device__ inline void device_lane_error(int64_t s, int code, int64_t a, int64_t b, int32_t* errors,
                                                  int64_t* info) {
  if (errors[s] != NNAB_LANE_OK) return;
  errors[s] = code;
  info[2 * s] = a;
  info[2 * s + 1] = b;
}

__host__ __device__ inline void device_pool_slot(int64_t s, int64_t slots, int64_t* counters, const int32_t* lengths,
                                                 const uint8_t* end_in, int32_t* errors, int64_t* info,
                                                 int32_t* counts, nnab_stream_lane* lanes, int64_t chunk, int K,
                                                 int hop, int pad, int pad_mode) {
  const int64_t received = counters[s], frames = counters[slots + s];
  const bool ended = counters[2 * slots + s] != 0;
  const int64_t n = lengths[s];
  const int end = end_in[s] != 0;
  nnab_stream_lane ln{};
  ln.slot = s;
  int64_t T = 0;
  int code = NNAB_LANE_OK;
  StreamStep st{};
  if (n < 0 || n > chunk) {
    code = NNAB_LANE_ELENGTH;
  } else if (ended && (n > 0 || end)) {
    code = NNAB_LANE_EENDED;
  } else if (n > 0 || end) {
    const int64_t n_carry = received - chunk_carry_start(received, frames, hop, pad);
    if (stream_step(received, n_carry, frames, n, end, K, hop, pad, pad_mode, &st) != NNAB_OK) {
      code = NNAB_LANE_ESHORT;  // the counters are the plan's own: only the end can be refused
    } else {
      ln.received = received; ln.n_carry = n_carry; ln.frames = frames; ln.n = n; ln.end = end;
      T = st.T;
      counters[s] = st.total;
      counters[slots + s] = st.t_end;
      counters[2 * slots + s] = ended || end;
    }
  }
  if (code != NNAB_LANE_OK)
    device_lane_error(s, code, code == NNAB_LANE_ESHORT ? received + n : n, 0, errors, info);
  lanes[s] = ln;
  counts[s] = (int32_t)T;
}

// device_pool_slot for a pool of pyramid streams: the counters' n_carry is the raw ring's (pyr_keep of signal 0),
// the rules pyr_step's.  The counters are the plan's own, so only an end can be refused (NNAB_LANE_ESHORT, info:
// the stream's length): pyr_stream_init's ring bounds hold every push that does not end.
__host__ __device__ inline void device_pyramid_slot(int64_t s, int64_t slots, int64_t* counters,
                                                    const int32_t* lengths, const uint8_t* end_in, int32_t* errors,
                                                    int64_t* info, int32_t* counts, nnab_stream_lane* lanes,
                                                    int64_t chunk, const PyrStream& p, int pad_mode) {
  const int64_t received = counters[s], frames = counters[slots + s];
  const bool ended = counters[2 * slots + s] != 0;
  const int64_t n = lengths[s];
  const int end = end_in[s] != 0;
  nnab_stream_lane ln{};
  ln.slot = s;
  int64_t T = 0;
  int code = NNAB_LANE_OK;
  if (n < 0 || n > chunk) {
    code = NNAB_LANE_ELENGTH;
  } else if (ended && (n > 0 || end)) {
    code = NNAB_LANE_EENDED;
  } else if (n > 0 || end) {
    PyrStep st;
    pyr_counts(p, received, 0, st.R0);
    const int64_t n_carry = received - pyr_keep(p, 0, st.R0, frames);
    if (pyr_step(p, received, n_carry, frames, n, end, pad_mode, &st) != NNAB_OK) {
      code = NNAB_LANE_ESHORT;
    } else {
      ln.received = received; ln.n_carry = n_carry; ln.frames = frames; ln.n = n; ln.end = end;
      T = st.t_end - frames;
      counters[s] = received + n;
      counters[slots + s] = st.t_end;
      counters[2 * slots + s] = ended || end;
    }
  }
  if (code != NNAB_LANE_OK)
    device_lane_error(s, code, code == NNAB_LANE_ESHORT ? received + n : n, 0, errors, info);
  lanes[s] = ln;
  counts[s] = (int32_t)T;
}

__host__ __device__ inline void device_istft_slot(int64_t s, int64_t slots, int64_t* counters,
                                                  const int32_t* frame_counts, const uint8_t* end_in,
                                                  const int64_t* length_in, int32_t* errors, int64_t* info,
                                                  int32_t* counts, nnab_istft_lane* lanes, int64_t t, int n_fft,
                                                  int hop, int center) {
  const int64_t frames = counters[s], emitted = counters[slots + s];
  const bool ended = counters[2 * slots + s] != 0;
  const int64_t T = frame_counts[s];
  const int end = end_in[s] != 0;
  const int64_t length = end ? (length_in[s] < 0 ? -1 : length_in[s]) : -1;
  nnab_istft_lane ln{};
  ln.slot = s; ln.row = -1; ln.length = -1;
  int64_t n_out = 0;
  int code = NNAB_LANE_OK;
  IstftChunkPlan pl{};
  if (T < 0 || T > t) {
    code = NNAB_LANE_ELENGTH;
  } else if (ended && (T > 0 || end)) {
    code = NNAB_LANE_EENDED;
  } else if (end && frames + T == 0) {
    code = NNAB_LANE_ENOFRAMES;
  } else if (T > 0 || end) {
    if (istft_chunk_plan(frames, emitted, T, n_fft, hop, center, end, length, &pl) != NNAB_OK) {
      code = NNAB_LANE_ELENGTH_SHORT;  // the counters are the plan's own: only the length can be refused
    } else {
      ln.row = T > 0 ? s : -1; ln.frames = frames; ln.emitted = emitted; ln.T = T; ln.end = end; ln.length = length;
      n_out = pl.emit_end - pl.emit_begin;
      counters[s] = frames + T;
      counters[slots + s] = emitted + n_out;
      counters[2 * slots + s] = ended || end;
    }
  }
  if (code != NNAB_LANE_OK)
    device_lane_error(s, code, code == NNAB_LANE_ELENGTH_SHORT ? length : T, emitted, errors, info);
  lanes[s] = ln;
  counts[s] = (int32_t)n_out;
}

struct FramedProblem {
  const void* x;       // (B, L) rows, pitch x_pitch samples of type x_dtype
  int x_dtype;         // NNAB_DTYPE_*: only the pad / split pre-pass reads 16-bit samples, the SIMT kernel fp32
  int64_t B, L, x_pitch;
  const float* w_re;   // (F, K)
  const float* w_im;   // (F, K)
  int F, K, hop;
  int pad;             // samples of centre padding on each side (0 if !center)
  int pad_mode;        // NNAB_PAD_*
  const float* scale;  // per-bin or nullptr
  float scale_all;
  int fmt;
  float eps;
  float power;         // FMT_POWER only
  float* out;
  int64_t T;
  int out_bins;        // rows of the output tensor (>= bins written)
  int bin_offset;      // output row of bin 0 (may be negative: rows < 0 dropped)
  const int32_t* h_k_begin;  // host, per-bin support or nullptr
  const int32_t* h_k_end;
  const FbEntry* fb_table;   // FMT_FBANK: device table [F]; out is (B, n_fb, T), pre-zeroed
  const FbStep* fb_steps;    // FMT_FBANK, block-partial kernel: [F + FB_STEP_PAD] (nullptr: MelRun path)
  int fb_nb_mask;            // bit i: tile width nb = 32 + 8 i gives <= 2 partial sums per filter
  int fb_poly_tile;          // four-phase block kernel: the cheapest nb giving <= 2 partial sums, or 0
  int n_fb;
  float* raw;                // tensor-core split-K scratch: 2 planes (re, im) of B*F*T floats, or nullptr
  const void* presplit;      // tensor-core path: already padded + split signal planes (skip pad_split)
  int64_t presplit_t_slots;  // > 0: frames per clip slot of the pre-split planes (else derived)
  int64_t presplit_plane_stride;  // elements per plane when presplit_t_slots > 0
  DecimParams dec;           // FMT_DECIM
  int64_t ola_pitch;         // FMT_OLA: out = overlap-add buffer (B, ola_pitch); scale = window/n_fft
  int ola_hop;
  int k_splits_hint;         // FMT_OLA only (its atomics already accumulate): cut K into chunks
  int64_t planes_stride;     // FMT_PLANES: elements between the hi and the lo plane
  int planes_pitch;          // FMT_PLANES: elements per frame row (multiple of 64)
  // non-null: the tensor-core pre-pass builds the planes from this push's virtual clip instead of x
  // (then L = chunk->length, pad = 0); the SIMT kernel returns NNAB_EUNSUPPORTED
  const ChunkSource* chunk;
  // host, or nullptr: receives the NNAB_CQ1992_* kernel route a successful launch enqueued (ROUTE_BLOCK for the
  // block-partial kernel, which only the STFT family runs)
  int* route;
};
constexpr int ROUTE_BLOCK = NNAB_CQ1992_ROUTES;

int launch_framed_simt(const FramedProblem& p, cudaStream_t stream);

// tensor-core path (tc_kernels.cu)
// packed: the basis the launch will use, when known (a block-partial basis has its own shape limits)
bool tc_supported(const FramedProblem& p, const void* packed = nullptr);
size_t tc_workspace_bytes(int64_t B, int64_t L, int K, int hop, int pad);
int launch_framed_tc(const FramedProblem& p, const void* packed, void* workspace,
                     size_t ws_bytes, cudaStream_t stream);
size_t tc_packed_bytes(int F, int K);
int tc_pack_basis(const float* w_re, const float* w_im, int F, int K, void* packed,
                  cudaStream_t stream);
int tc_tile_n(int F);
int tc_pack_basis_layout(const float* w_re, const float* w_im, int F, int K, int layout, void* packed,
                         cudaStream_t stream);
// split-signal geometry / helpers for callers that manage the planes themselves (pyramid)
void tc_split_geometry(int64_t B, int64_t L, int K, int hop, int pad, int64_t* t_slots,
                       int64_t* plane_stride, int* hop_eff);
// (x: samples of type x_dtype, NNAB_DTYPE_*; the planes equal those of the samples converted to fp32)
int tc_pad_split(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch, int K, int hop, int pad,
                 int pad_mode, void* planes, cudaStream_t stream);
int tc_pad_split_ex(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch, int pad, int pad_mode,
                    int64_t clip_pitch, int64_t plane_stride, void* planes, cudaStream_t stream);
// tc_pad_split on the problem's own signal: the waveform x with its centre padding, or a push's virtual clip.
// TC_SPLIT_POLY4 (hop % 128 == 0) stores every hop-sized block in polyphase order: position q * hop / 4 + m
// holds sample 4 m + q (the four-phase block-partial kernel reads the four phases as four K ranges).
constexpr int TC_SPLIT_PLAIN = 0;
constexpr int TC_SPLIT_POLY4 = 1;
int tc_problem_split(const FramedProblem& q, void* planes, cudaStream_t stream, int layout);
// planes of the B virtual clips of cs, row b that of lane b (clip_pitch samples per clip from its first sample),
// in a caller geometry
int tc_chunk_split(const ChunkSource& cs, int x_dtype, int64_t B, int64_t clip_pitch, int64_t plane_stride,
                   void* planes, cudaStream_t stream);
// the carry of every one of the n_lanes lanes of cs (lanes[i], or `shared` in slot i): each stores its own raw
// samples [from, received + n) of the chunk into its ring row (at most `longest` samples); and for a lane table,
// the zeroing of output frames t >= the count of row i of out (A, rows, T, cols)
int tc_pool_carry(const ChunkSource& cs, int x_dtype, int64_t n_lanes, int64_t longest, cudaStream_t stream);
int tc_pool_mask(const ChunkSource& cs, int64_t A, float* out, int64_t rows, int64_t T, int cols,
                 cudaStream_t stream);
// device pools: the plan launches (device_pool_slot / device_istft_slot per slot) and the masked reset
int tc_device_pool_plan(int64_t slots, int64_t* counters, const int32_t* lengths, const uint8_t* end,
                        int32_t* errors, int64_t* info, int32_t* counts, nnab_stream_lane* lanes, int64_t chunk,
                        int K, int hop, int pad, int pad_mode, cudaStream_t stream);
int tc_device_istft_plan(int64_t slots, int64_t* counters, const int32_t* frame_counts, const uint8_t* end,
                         const int64_t* length, int32_t* errors, int64_t* info, int32_t* counts,
                         nnab_istft_lane* lanes, int64_t t, int n_fft, int hop, int center, cudaStream_t stream);
int tc_device_pool_reset(int64_t slots, int64_t* counters, int32_t* errors, int64_t* info, const uint8_t* mask,
                         cudaStream_t stream);

// ---- PCEN (pcen_kernels.cu) ---------------------------------------------------
// per-channel (param_stride 1) or scalar (0) parameters, device pointers
struct PcenArgs {
  const float *s, *gain, *bias, *power;
  int param_stride;
  float eps;
};
// the streamed call's state: state / primed (slots, C); row b is slot row_slot[b] (NULL: slot b) and advances by
// counts[b] frames (NULL: all of them); state == NULL for the offline and training calls
struct PcenStream {
  float* state;
  uint8_t* primed;
  int64_t slots;
  const int32_t* row_slot;
  const int32_t* counts;
};
int64_t pcen_blocks(int64_t rows);
int pcen_forward(const float* E, int64_t B, int C, int64_t T, const PcenArgs& a, float* P, float* M_out,
                 const PcenStream& st, cudaStream_t stream);
// partial: 4 * B * C floats of workspace when grad_params != NULL
int pcen_backward(const float* E, const float* M, const float* gP, int64_t B, int C, int64_t T, const PcenArgs& a,
                  float* dE, float* grad_params, float* partial, cudaStream_t stream);
int pcen_reset(uint8_t* primed, const uint8_t* mask, int64_t slots, int C, cudaStream_t stream);
// pyramid pools: the (signal, lane) descriptor table of a push (table[s * n_lanes + i] = pyr_lane_signal of lane i
// of the DEVICE lane table, or with lanes == nullptr of `shared` in slot i), every row's carry [keep, R1) of one
// signal (cs.rows; at most `longest` samples), and the zeroing of frames t >= rows[i].count of row i of out
// (A, n_rows, T, cols)
int tc_pyr_pool_plan(const PyrStream& p, const nnab_stream_lane* lanes, const nnab_stream_lane& shared,
                     int64_t n_lanes, int pad_mode, PyrLaneSig* table, cudaStream_t stream);
// device pyramid pools: the plan launch (device_pyramid_slot per slot)
int tc_device_pyramid_plan(const PyrStream& p, int64_t slots, int64_t* counters, const int32_t* lengths,
                           const uint8_t* end, int32_t* errors, int64_t* info, int32_t* counts,
                           nnab_stream_lane* lanes, int64_t chunk, int pad_mode, cudaStream_t stream);
int tc_rows_carry(const ChunkSource& cs, int x_dtype, int64_t n_rows, int64_t longest, cudaStream_t stream);
int tc_rows_mask(const PyrLaneSig* rows, int64_t A, float* out, int64_t n_rows, int64_t T, int cols,
                 cudaStream_t stream);
int tc_zero_slots(void* planes, int64_t B, int64_t clip_pitch, int64_t plane_stride, int64_t keep_lo,
                  int64_t keep_hi, cudaStream_t stream);
int tc_pad_split2(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch,
                  int K_a, int hop_a, int pad_a, int mode_a, void* planes_a,
                  int K_b, int hop_b, int pad_b, int mode_b, void* planes_b, cudaStream_t stream);
// inverse STFT pieces (tc_kernels.cu)
int tc_istft_k(int f_in);
int tc_istft_bn(int n_fft);
// Launch shape of the FMT_OLA GEMM (the inverse STFT and both gradients): M_rows frames (rows) x F_out output
// samples in n_tiles tiles of bn, K_gemm rounded up to 64 and cut into k_splits chunks of at most 64 k-blocks (at
// most k_splits_hint of them), exec_flops the MMA flops of the launch.  tc_supported and launch_framed_tc both read it.
struct OlaPlan {
  int supported, bn, n_tiles, k_splits;
  double exec_flops;
};
OlaPlan tc_ola_plan(int F_out, int K_gemm, int64_t M_rows, int k_splits_hint);
constexpr int TC_OLA_MAX_SPLITS = 64;  // the K chunks the offline callers allow
size_t tc_packed_istft_bytes(int n_fft, int f_in);
int tc_pack_istft(const float* kc, const float* ks, int n_fft, int f_in, int onesided, void* packed,
                  cudaStream_t stream, int transposed = 0);
// weight-gradient operands (tc_kernels.cu)
int64_t tc_dw_gpad(int64_t B, int64_t T);
size_t tc_dw_grad_planes_bytes(int64_t B, int64_t T, int F);
size_t tc_dw_frames_bytes(int64_t B, int64_t T, int K);
int tc_dw_prep_grad(const float* g, int64_t B, int F, int64_t T, void* planes, cudaStream_t stream);
int tc_dw_prep_frames(const float* x, int64_t B, int64_t L, int64_t x_pitch, int K, int hop, int pad,
                      int pad_mode, int64_t T, void* packed, cudaStream_t stream);
int tc_unpad_adjoint(const float* gp, int64_t gp_pitch, int64_t gp_len, int64_t B, int pad,
                     int pad_mode, int64_t L, float* dx, cudaStream_t stream);
size_t tc_istft_planes_bytes(int64_t B, int64_t T, int f_in);
int tc_istft_prep(const float* X, int64_t B, int f_in, int64_t T, void* planes, cudaStream_t stream);
int tc_istft_finalize(const float* ola, int64_t ola_pitch, int64_t B, const float* window,
                      int n_fft, int hop, int64_t T, int64_t offset, float* out, int64_t out_len,
                      cudaStream_t stream);
// inverse STFT pools: lane i is lanes[i] of the DEVICE lane table or, without one (a lock-step push), `shared` in
// slot i.  Row i of the (n_lanes, ola_pitch) overlap-add buffer holds lane i's positions from frames_i * hop - lead.
// Seed: every row's carried sums from its state row, zeros elsewhere.  Prep: plane row i * T_max + t from
// X[row_i, :, t] of the (R, f_in, x_T, 2) frames for t < T_i, zeros past T_i and for row_i = -1 (without a lane
// table, X is (n_lanes, f_in, T_max, 2)).  Finalize: rows i < A of out (A, n_max) get lane i's final samples then
// zeros; every lane's open tail goes to its state row.
int tc_istft_pool_seed(const nnab_istft_lane* lanes, const nnab_istft_lane& shared, int64_t n_lanes,
                       const float* state, int n_fft, int hop, int center, int64_t lead, float* ola, int64_t ola_pitch,
                       cudaStream_t stream);
int tc_istft_pool_prep(const float* X, const nnab_istft_lane* lanes, int64_t n_lanes, int f_in, int64_t T_max,
                       int64_t x_T, void* planes, cudaStream_t stream);
int tc_istft_pool_finalize(const nnab_istft_lane* lanes, const nnab_istft_lane& shared, int64_t n_lanes, int64_t A,
                           const float* ola, int64_t ola_pitch, int64_t lead, const float* window, int n_fft, int hop,
                           int center, float* out, int64_t n_max, float* state, cudaStream_t stream);
size_t tc_splitk_scratch_bytes(int64_t B, int F, int64_t T, int K);
// block-partial kernel (tcb_kernels.cu): default N-tile geometry of an (n_fft, hop) transform (nb packed
// columns per tile, nb - 2 new bins each, `phases` families per tile: 1, or 4 when hop % 128 == 0) -- the column
// layout of the FMT_PLANES operand planes: tile n, family f at columns nb (phases n + f) ..
void tc_block_tile_geometry(int n_fft, int hop, int* nb, int* n_tiles, int* phases);
bool tc_block_shape_ok(int n_fft, int hop);
size_t tc_packed_fir_bytes(int taps, int dec);
int tc_fir_k(int taps, int dec);
int tc_pack_fir(const float* fir, int taps, int dec, void* packed, cudaStream_t stream);
int launch_fb_table(const float* fb, int n_fb, int F, FbEntry* table, int* d_max_nnz,
                    cudaStream_t stream);
// FbEntry[F] -> FbStep[F + FB_STEP_PAD]; d_meta[0] = widest filter support (bins), d_meta[1] = bit mask
// of the tile widths nb = 32 + 8 i under which every filter gets <= 2 partial sums in the one-phase block
// kernel, d_meta[2] = the cheapest nb that does so in the four-phase kernel, or 0
int launch_fb_steps(const FbEntry* table, int n_fb, int F, FbStep* steps, int* d_meta,
                    cudaStream_t stream);

// filterbank / MFCC tail / FIR decimation (simt_kernels.cu)
int launch_filterbank(const float* P, const float* fb, int64_t B, int F, int64_t T, int n_fb,
                      float* out, cudaStream_t stream);
int launch_fb_tile_bank(const float* fb, int n_fb, int F, int nb, int n_tiles, int phases, int kp, int fh, float* w_re,
                        float* w_im, cudaStream_t stream);
// clip_max_kernel puts one clip on each blockIdx.y
constexpr int64_t MFCC_MAX_CLIPS = 65535;
int launch_mfcc_tail(const float* mel, int64_t B, int n_mels, int64_t T, float amin, float ref,
                     float top_db, const float* dct, int n_mfcc, float* out,
                     unsigned int* scratch /* B words */, cudaStream_t stream);
int tc_varn_plan_export(const int32_t* k_begin, const int32_t* k_end, int F, int K, int want_chunks,
                        int32_t* order, int32_t* groups, int32_t* chunk_begin, int32_t* n_blocks,
                        int32_t* n_chunks);
int launch_fir_decimate_adjoint(const float* g, int64_t B, int64_t T, int64_t g_pitch,
                                const float* fir, int taps, int factor, float* dx, int64_t L,
                                int64_t dx_pitch, cudaStream_t stream);
int launch_fir_decimate(const float* x, int64_t B, int64_t L, int64_t x_pitch, const float* fir,
                        int taps, int factor, float* y, int64_t Ly, int64_t y_pitch,
                        cudaStream_t stream);

inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

}  // namespace nnab
