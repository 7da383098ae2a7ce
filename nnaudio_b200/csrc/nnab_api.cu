// extern "C" entry points of libnnab.so — see include/nnab.h for the contract
// and the reference file:line each call replaces.
#include <cuda.h>
#include <cuda_bf16.h>
#include <algorithm>
#include <atomic>
#include <climits>
#include <mutex>
#include <stdlib.h>
#include <string.h>
#include <unordered_map>
#include <utility>
#include <vector>

#include "common.cuh"
#include "tc_host.cuh"

namespace nnab {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};
static std::atomic<uint64_t> g_balanced_launches{0};
static std::atomic<uint64_t> g_block_ws_launches{0};

void set_cuda_error(const char* where, cudaError_t e) {
  snprintf(g_err, sizeof(g_err), "%s: %s (%s)", where, cudaGetErrorName(e), cudaGetErrorString(e));
}
void set_error_text(const char* text) { snprintf(g_err, sizeof(g_err), "%s", text); }
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
void count_balanced_launch() { g_balanced_launches.fetch_add(1, std::memory_order_relaxed); }
void count_block_ws_launch() { g_block_ws_launches.fetch_add(1, std::memory_order_relaxed); }
static std::atomic<uint64_t> g_pyr_routes[NNAB_PYR_ROUTES];
static void count_route(int route) { g_pyr_routes[route].fetch_add(1, std::memory_order_relaxed); }
static std::atomic<uint64_t> g_cq1992_routes[NNAB_CQ1992_ROUTES];
static std::atomic<uint64_t> g_stft_routes[NNAB_STFT_ROUTES];
// the same routes, counted by the chunk, pool and device-pool entry points (nnab_stream_route_count)
static std::atomic<uint64_t> g_stream_stft[NNAB_STFT_ROUTES];
static std::atomic<uint64_t> g_stream_cq1992[NNAB_CQ1992_ROUTES];
static std::atomic<uint64_t> g_stream_pyr[NNAB_PYR_ROUTES];
// routes[0]: the contraction's kernel route (NNAB_CQ1992_* / ROUTE_BLOCK, as the launchers write it); routes[1]:
// the filterbank route (NNAB_STFT_FB_*), or -1
static void count_stft_routes(const int (&routes)[2], std::atomic<uint64_t>* counters = g_stft_routes) {
  int r = -1;
  switch (routes[0]) {
    case ROUTE_BLOCK: r = NNAB_STFT_BLOCK; break;
    case NNAB_CQ1992_DENSE: r = NNAB_STFT_DENSE; break;
    case NNAB_CQ1992_DENSE_SPLITK: r = NNAB_STFT_DENSE_SPLITK; break;
    case NNAB_CQ1992_SIMT: r = NNAB_STFT_SIMT; break;
  }
  if (r >= 0) counters[r].fetch_add(1, std::memory_order_relaxed);
  if (routes[1] >= 0) counters[routes[1]].fetch_add(1, std::memory_order_relaxed);
}
static void count_cq1992_route(int route, std::atomic<uint64_t>* counters) {
  if (route >= 0) counters[route].fetch_add(1, std::memory_order_relaxed);
}
static std::atomic<int> g_sm_reserve{0};
int sm_reserve() { return g_sm_reserve.load(std::memory_order_relaxed); }
// persistent-grid ledger (nnab_persistent_grid_read): launches, summed CTAs, min and max grid since the last read
static std::atomic<uint64_t> g_pgrid_launches{0};
static std::atomic<uint64_t> g_pgrid_ctas{0};
static std::atomic<int> g_pgrid_min{INT_MAX};
static std::atomic<int> g_pgrid_max{0};
void count_persistent_grid(int grid) {
  g_pgrid_launches.fetch_add(1, std::memory_order_relaxed);
  g_pgrid_ctas.fetch_add((uint64_t)grid, std::memory_order_relaxed);
  int lo = g_pgrid_min.load(std::memory_order_relaxed);
  while (grid < lo && !g_pgrid_min.compare_exchange_weak(lo, grid, std::memory_order_relaxed)) {
  }
  int hi = g_pgrid_max.load(std::memory_order_relaxed);
  while (grid > hi && !g_pgrid_max.compare_exchange_weak(hi, grid, std::memory_order_relaxed)) {
  }
}

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// T of a centred / un-centred framing: (L + 2*pad - K)/hop + 1
static inline int64_t frames_of(int64_t L, int K, int hop, int pad) {
  const int64_t span = L + 2 * (int64_t)pad - K;
  return span < 0 ? 0 : span / hop + 1;
}

static bool dtype_ok(int x_dtype) {
  return x_dtype == NNAB_DTYPE_F32 || x_dtype == NNAB_DTYPE_BF16 || x_dtype == NNAB_DTYPE_F16;
}

static int check_common(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch, int K, int F,
                        int hop, int pad, int pad_mode, int64_t T) {
  if (x == nullptr || !dtype_ok(x_dtype) || B < 0 || L <= 0 || x_pitch < L || K <= 0 || F <= 0 || hop <= 0)
    return NNAB_EINVAL;
  if (pad_mode != NNAB_PAD_REFLECT && pad_mode != NNAB_PAD_CONSTANT) return NNAB_EINVAL;
  // nn.ReflectionPad1d needs pad < L; callers raise the reference's exception first.
  if (pad > 0 && pad_mode == NNAB_PAD_REFLECT && pad >= L) return NNAB_EINVAL;
  if (T != frames_of(L, K, hop, pad) || T <= 0) return NNAB_EINVAL;
  return NNAB_OK;
}

static int check_arch() {
  int dev = 0;
  NNAB_CUDA_TRY(cudaGetDevice(&dev));
  int major = 0, minor = 0;
  NNAB_CUDA_TRY(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  NNAB_CUDA_TRY(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  return (major == 9 && minor == 0) ? NNAB_OK : NNAB_EARCH;  // sm_90a code runs on compute capability 9.0 only
}

// ---- optional in-stream timing of the framed contraction (bench.py) --------
static std::atomic<int> g_prof_on{0};
static std::mutex g_prof_mu;
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_pairs;  // recorded, unread
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_free;

static double g_exec_flops = 0.0;  // guarded by g_prof_mu
void add_exec_flops(double flops) {
  if (!g_prof_on.load(std::memory_order_relaxed)) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_exec_flops += flops;
}

static bool prof_begin(cudaStream_t s, std::pair<cudaEvent_t, cudaEvent_t>* pr) {
  if (!g_prof_on.load(std::memory_order_relaxed)) return false;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (!g_prof_free.empty()) {
    *pr = g_prof_free.back();
    g_prof_free.pop_back();
  } else {
    if (cudaEventCreate(&pr->first) != cudaSuccess) return false;
    if (cudaEventCreate(&pr->second) != cudaSuccess) return false;
  }
  cudaEventRecord(pr->first, s);
  return true;
}
static void prof_end(cudaStream_t s, const std::pair<cudaEvent_t, cudaEvent_t>& pr) {
  cudaEventRecord(pr.second, s);
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof_pairs.push_back(pr);
}

static int run_framed_inner(const FramedProblem& p, const void* packed, void* ws, size_t ws_bytes,
                            int path, cudaStream_t stream);

// Run one framed contraction on the requested kernel family.
static int run_framed(const FramedProblem& p, const void* packed, void* ws, size_t ws_bytes,
                      int path, cudaStream_t stream) {
  std::pair<cudaEvent_t, cudaEvent_t> pr;
  const bool timed = prof_begin(stream, &pr);
  const int rc = run_framed_inner(p, packed, ws, ws_bytes, path, stream);
  if (timed) prof_end(stream, pr);
  return rc;
}

static int run_framed_inner(const FramedProblem& p, const void* packed, void* ws, size_t ws_bytes,
                      int path, cudaStream_t stream) {
  bool use_tc = false;
  if (path == NNAB_PATH_TCGEN05) {
    if (packed == nullptr || !tc_supported(p, packed)) return NNAB_EALIGN;
    use_tc = true;
  } else if (path == NNAB_PATH_AUTO) {
    use_tc = (packed != nullptr) && tc_supported(p, packed);
  } else if (path != NNAB_PATH_SIMT) {
    return NNAB_EINVAL;
  }
  if (use_tc) return launch_framed_tc(p, packed, ws, ws_bytes, stream);
  const int rc = launch_framed_simt(p, stream);
  if (rc == NNAB_OK && p.route != nullptr) *p.route = NNAB_CQ1992_SIMT;
  return rc;
}

// The split-K scratch (long kernels only) sits behind the split-signal planes in the workspace.
static void attach_splitk_scratch(FramedProblem& p, void* workspace, size_t ws_bytes) {
  const size_t sk = tc_splitk_scratch_bytes(p.B, p.F, p.T, p.K);
  if (sk == 0 || workspace == nullptr) return;
  const size_t front = align_up(tc_workspace_bytes(p.B, p.L, p.K, p.hop, p.pad), 256);
  if (front + sk <= ws_bytes) p.raw = reinterpret_cast<float*>((char*)workspace + front);
}

static bool wants_tc(int path, int K, int hop) {
  if (path == NNAB_PATH_SIMT) return false;
  FramedProblem q{};
  q.K = K; q.hop = hop; q.F = 1; q.B = 1; q.L = K; q.T = 1;
  return tc_supported(q);
}

// The signal a forward call's framed problems read: the caller's waveform with its centre padding, or one
// push's virtual clip (chunk != nullptr; then L is the clip's length and pad 0).
struct Wave {
  const void* x;
  int x_dtype;
  int64_t B, L, x_pitch;
  int pad, pad_mode;
  const ChunkSource* chunk;
};

static void set_wave(FramedProblem& p, const Wave& w) {
  p.x = w.x; p.x_dtype = w.x_dtype; p.B = w.B; p.L = w.L; p.x_pitch = w.x_pitch;
  p.pad = w.pad; p.pad_mode = w.pad_mode; p.chunk = w.chunk;
}

// ---- chunked streams and stream pools (DESIGN §3.10) ----------------------------------------------------
// A push of lanes, each one stream (counters: StreamStep / stream_step in common.cuh).  A pool's lanes come from
// its device lane table; a lock-step push of B streams is the push of B lanes that share one set of counters.
struct PoolPlan {
  ChunkSource cs;     // lanes = the device table, or nullptr and `shared`; length = the clip of T_max frames
  int64_t A, T_max;
  int64_t longest;    // the most samples one lane stores into the ring
};

// The source of a push's clips of `length` samples: ring rows of K floats, chunk rows of chunk_pitch samples.
static ChunkSource chunk_source(const void* state, const void* chunk, int64_t chunk_pitch, int K, int hop, int pad,
                                int pad_mode, int64_t length, const nnab_stream_lane* lanes,
                                const nnab_stream_lane& shared) {
  ChunkSource c{};
  c.ring = static_cast<const float*>(state);
  c.ring_pitch = K;
  c.ring_len = K;
  c.chunk = chunk;
  c.chunk_pitch = chunk_pitch;
  c.length = length;
  c.pad_mode = pad > 0 ? pad_mode : NNAB_PAD_CONSTANT;
  c.lanes = lanes;
  c.shared = shared;
  c.K = K; c.hop = hop; c.pad = pad;
  return c;
}

// A lock-step push: B streams with these counters, lane b in slot b; T_max is the frames it returns.
static int lock_step_plan(const void* state, int64_t received, int64_t n_carry, int64_t frames, const void* chunk,
                          int chunk_dtype, int64_t B, int64_t n, int64_t chunk_pitch, int flush, int K, int hop,
                          int pad, int pad_mode, PoolPlan* o) {
  if (state == nullptr || !dtype_ok(chunk_dtype) || B < 0 || B > 65535 || n < 0 || (n > 0 && chunk == nullptr) ||
      chunk_pitch < n || K < 2 || hop <= 0)
    return NNAB_EINVAL;
  if (pad_mode != NNAB_PAD_REFLECT && pad_mode != NNAB_PAD_CONSTANT) return NNAB_EINVAL;
  StreamStep st;
  const int rc = stream_step(received, n_carry, frames, n, flush, K, hop, pad, pad_mode, &st);
  if (rc) return rc;
  const nnab_stream_lane ln{0, received, n_carry, frames, n, flush ? 1 : 0};
  o->cs = chunk_source(state, chunk, chunk_pitch, K, hop, pad, pad_mode, st.T > 0 ? (st.T - 1) * hop + K : 0,
                       nullptr, ln);
  o->A = st.T > 0 ? B : 0;
  o->T_max = st.T;
  o->longest = st.total - st.from;
  return NNAB_OK;
}

// Checks the whole push (every lane by stream_step, the table's order and totals) before anything runs.
static int pool_plan(const void* state, const nnab_stream_lane* lanes, const nnab_stream_lane* d_lanes,
                     int64_t n_lanes, int64_t A, const void* chunk, int chunk_dtype, int64_t slots, int64_t n,
                     int64_t chunk_pitch, int K, int hop, int pad, int pad_mode, int64_t T_max, PoolPlan* o) {
  if (state == nullptr || !dtype_ok(chunk_dtype) || slots < 1 || slots > 65535 || n < 0 ||
      (n > 0 && chunk == nullptr) || chunk_pitch < n || K < 2 || hop <= 0 || n_lanes < 0 || n_lanes > slots ||
      A < 0 || A > n_lanes || T_max < 0 || (n_lanes > 0 && (lanes == nullptr || d_lanes == nullptr)))
    return NNAB_EINVAL;
  if (pad_mode != NNAB_PAD_REFLECT && pad_mode != NNAB_PAD_CONSTANT) return NNAB_EINVAL;
  std::vector<uint8_t> seen((size_t)slots, 0);
  int64_t t_max = 0, longest = 0;
  for (int64_t i = 0; i < n_lanes; ++i) {
    const nnab_stream_lane& ln = lanes[i];
    if (ln.slot < 0 || ln.slot >= slots || seen[(size_t)ln.slot]) return NNAB_EINVAL;
    if (i > 0 && i != A && ln.slot <= lanes[i - 1].slot) return NNAB_EINVAL;  // ascending within each group
    seen[(size_t)ln.slot] = 1;
    if (ln.n > n || (ln.end != 0 && ln.end != 1)) return NNAB_EINVAL;
    StreamStep st;
    const int rc = stream_step(ln.received, ln.n_carry, ln.frames, ln.n, (int)ln.end, K, hop, pad, pad_mode, &st);
    if (rc) return rc;
    if ((i < A) != (st.T > 0)) return NNAB_EINVAL;           // the A lanes with frames come first
    if (st.T == 0 && ln.n == 0 && !ln.end) return NNAB_EINVAL;  // a lane with nothing to do
    if (st.T > t_max) t_max = st.T;
    if (st.total - st.from > longest) longest = st.total - st.from;
  }
  if (t_max != T_max) return NNAB_EINVAL;
  o->cs = chunk_source(state, chunk, chunk_pitch, K, hop, pad, pad_mode, T_max > 0 ? (T_max - 1) * hop + K : 0,
                       d_lanes, nnab_stream_lane{});
  o->A = A;
  o->T_max = T_max;
  o->longest = longest;
  return NNAB_OK;
}

// Floats per (row, frame) of an output format (nnab.h): complex pairs and unit phasors take two.
static int format_cols(int out_format) {
  return out_format == NNAB_FMT_COMPLEX || out_format == NNAB_FMT_PHASE_UNIT ? 2 : 1;
}

// Clip length of a pool push's batch (0: no lane returns a frame); host only, no validation.
static int64_t pool_clip_length(int64_t A, int64_t T_max, int K, int hop) {
  return A > 0 && T_max > 0 ? (T_max - 1) * (int64_t)hop + K : 0;
}

// The offline plan on the A rows' clips, the zeroing of every row's frames past its count, then each lane's
// carry.  A plan that cannot read the clips (the SIMT kernels) returns NNAB_EUNSUPPORTED before anything is
// enqueued, the ring included (when A > 0).  Lanes that share their counters all return T_max frames: nothing
// to zero.
template <typename Run>
static int pool_forward(const PoolPlan& pp, int chunk_dtype, int64_t n_lanes, float* out, int64_t rows, int cols,
                        Run&& run, void* stream) {
  int rc = check_arch();
  if (rc) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  if (pp.A > 0) {
    const Wave w{nullptr, chunk_dtype, pp.A, pp.cs.length, pp.cs.length, 0, pp.cs.pad_mode, &pp.cs};
    if ((rc = run(w, s))) return rc;
    if (pp.cs.lanes != nullptr && (rc = tc_pool_mask(pp.cs, pp.A, out, rows, pp.T_max, cols, s))) return rc;
  }
  return tc_pool_carry(pp.cs, chunk_dtype, n_lanes, pp.longest, s);
}

// The host-side checks of a device-planned push and its fixed geometry: every slot is a lane (A = slots), each
// clip T_max = T_cap frames long, and a lane stores at most the chunk width into its ring.
static int device_pool_plan(void* state, int64_t* counters, const int32_t* lengths, const uint8_t* end,
                            int32_t* errors, int64_t* info, int32_t* counts, nnab_stream_lane* d_lanes,
                            const void* chunk, int chunk_dtype, int64_t slots, int64_t n, int64_t chunk_pitch, int K,
                            int hop, int pad, int pad_mode, int64_t T_max, float* out, PoolPlan* o) {
  if (state == nullptr || counters == nullptr || lengths == nullptr || end == nullptr || errors == nullptr ||
      info == nullptr || counts == nullptr || d_lanes == nullptr || chunk == nullptr || out == nullptr ||
      !dtype_ok(chunk_dtype) || slots < 1 || slots > 65535 || n < 1 || chunk_pitch < n || K < 2 || hop <= 0)
    return NNAB_EINVAL;
  if (pad_mode != NNAB_PAD_REFLECT && pad_mode != NNAB_PAD_CONSTANT) return NNAB_EINVAL;
  if (T_max != nnab_pool_frame_cap(n, K, hop, pad, pad_mode)) return NNAB_EINVAL;
  o->cs = chunk_source(state, chunk, chunk_pitch, K, hop, pad, pad_mode, (T_max - 1) * hop + K, d_lanes,
                       nnab_stream_lane{});
  o->A = slots;
  o->T_max = T_max;
  o->longest = n;
  return NNAB_OK;
}

// The plan launch, then the stream pools' body on every slot.
template <typename Run>
static int device_pool_forward(const PoolPlan& pp, int64_t* counters, const int32_t* lengths, const uint8_t* end,
                               int32_t* errors, int64_t* info, int32_t* counts, int chunk_dtype, int64_t n, float* out,
                               int64_t rows, int cols, Run&& run, void* stream) {
  int rc = check_arch();
  if (rc) return rc;
  const int pad_mode = pp.cs.pad_mode;
  if ((rc = tc_device_pool_plan(pp.A, counters, lengths, end, errors, info, counts,
                                const_cast<nnab_stream_lane*>(pp.cs.lanes), n, pp.cs.K, pp.cs.hop, pp.cs.pad, pad_mode,
                                (cudaStream_t)stream)))
    return rc;
  return pool_forward(pp, chunk_dtype, pp.A, out, rows, cols, run, stream);
}

// Frames a lock-step push returns (0: none); host only, no validation.
static int64_t chunk_frames(int64_t received, int64_t frames, int64_t n, int flush, int K, int hop, int pad,
                            int pad_mode) {
  const int64_t total = received + n;
  const int64_t t_end = flush ? frames_of(total, K, hop, pad) : chunk_ready_frames(total, K, hop, pad, pad_mode);
  return t_end > frames ? t_end - frames : 0;
}

// ---- streamed inverse STFT: istft_chunk_plan (common.cuh) ------------------------------------------

}  // namespace nnab

using namespace nnab;

extern "C" {

int nnab_abi_version(void) { return NNAB_ABI_VERSION; }

const char* nnab_strerror(int status) {
  switch (status) {
    case NNAB_OK: return "ok";
    case NNAB_EINVAL: return "invalid argument or shape mismatch";
    case NNAB_EALIGN: return "tensor-core path forced but shape/alignment rules not met";
    case NNAB_EARCH: return "device is not sm_90 (H100)";
    case NNAB_ECUDA: return "CUDA error";
    case NNAB_EWORKSPACE: return "workspace missing or too small";
    case NNAB_EUNSUPPORTED: return "unsupported size";
    default: return "unknown status";
  }
}

const char* nnab_last_cuda_error(void) { return g_err; }

uint64_t nnab_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

uint64_t nnab_balanced_launch_count(void) { return g_balanced_launches.load(std::memory_order_relaxed); }
uint64_t nnab_block_ws_launch_count(void) { return g_block_ws_launches.load(std::memory_order_relaxed); }
uint64_t nnab_pyramid_route_count(int route) {
  if (route < 0 || route >= NNAB_PYR_ROUTES) return 0;
  return g_pyr_routes[route].load(std::memory_order_relaxed);
}
uint64_t nnab_cqt1992v2_route_count(int route) {
  if (route < 0 || route >= NNAB_CQ1992_ROUTES) return 0;
  return g_cq1992_routes[route].load(std::memory_order_relaxed);
}
uint64_t nnab_stft_route_count(int route) {
  if (route < 0 || route >= NNAB_STFT_ROUTES) return 0;
  return g_stft_routes[route].load(std::memory_order_relaxed);
}
uint64_t nnab_stream_route_count(int family, int route) {
  switch (family) {
    case NNAB_ROUTES_STFT:
      return route < 0 || route >= NNAB_STFT_ROUTES ? 0 : g_stream_stft[route].load(std::memory_order_relaxed);
    case NNAB_ROUTES_CQ1992:
      return route < 0 || route >= NNAB_CQ1992_ROUTES ? 0 : g_stream_cq1992[route].load(std::memory_order_relaxed);
    case NNAB_ROUTES_PYR:
      return route < 0 || route >= NNAB_PYR_ROUTES ? 0 : g_stream_pyr[route].load(std::memory_order_relaxed);
  }
  return 0;
}

int nnab_set_sm_reserve(int n_sms) {
  if (n_sms < 0) n_sms = 0;
  return g_sm_reserve.exchange(n_sms);
}

int nnab_persistent_grid_read(uint64_t* launches, uint64_t* ctas, int* min_grid, int* max_grid) {
  const uint64_t n = g_pgrid_launches.exchange(0, std::memory_order_relaxed);
  const uint64_t c = g_pgrid_ctas.exchange(0, std::memory_order_relaxed);
  const int lo = g_pgrid_min.exchange(INT_MAX, std::memory_order_relaxed);
  const int hi = g_pgrid_max.exchange(0, std::memory_order_relaxed);
  if (launches) *launches = n;
  if (ctas) *ctas = c;
  if (min_grid) *min_grid = n ? lo : 0;
  if (max_grid) *max_grid = hi;
  return NNAB_OK;
}

void nnab_profile_enable(int on) { g_prof_on.store(on ? 1 : 0); }

int nnab_profile_read(double* framed_ms, uint64_t* framed_launches) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  double total = 0.0;
  uint64_t n = 0;
  for (auto& pr : g_prof_pairs) {
    NNAB_CUDA_TRY(cudaEventSynchronize(pr.second));
    float ms = 0.f;
    NNAB_CUDA_TRY(cudaEventElapsedTime(&ms, pr.first, pr.second));
    total += ms;
    ++n;
    g_prof_free.push_back(pr);
  }
  g_prof_pairs.clear();
  if (framed_ms) *framed_ms = total;
  if (framed_launches) *framed_launches = n;
  return NNAB_OK;
}

int nnab_profile_read_exec_flops(double* exec_flops) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (exec_flops) *exec_flops = g_exec_flops;
  g_exec_flops = 0.0;
  return NNAB_OK;
}

int nnab_pack_tile_n(int F) { return tc_tile_n(F); }
size_t nnab_packed_basis_bytes(int F, int K) { return tc_packed_bytes(F, K); }
int nnab_pack_basis(const float* w_re, const float* w_im, int F, int K, void* packed,
                    void* stream) {
  if (w_re == nullptr || w_im == nullptr || packed == nullptr || F <= 0 || K <= 0)
    return NNAB_EINVAL;
  return tc_pack_basis(w_re, w_im, F, K, packed, (cudaStream_t)stream);
}

int nnab_pack_basis_ex(const float* w_re, const float* w_im, int F, int K, int layout, void* packed,
                       void* stream) {
  if (w_re == nullptr || w_im == nullptr || packed == nullptr || F <= 0 || K <= 0)
    return NNAB_EINVAL;
  return tc_pack_basis_layout(w_re, w_im, F, K, layout, packed, (cudaStream_t)stream);
}

// Stream memory operations (multi-GPU gather handshakes without kernels): thin wrappers over the driver
// entry points, resolved at run time like cuTensorMapEncodeTiled.
typedef CUresult (*StreamValue32Fn)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
static StreamValue32Fn memop_fn(const char* name) {
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint(name, &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  return reinterpret_cast<StreamValue32Fn>(ptr);
}
int nnab_stream_write_value32(void* stream, void* addr, uint32_t value) {
  static StreamValue32Fn fn = memop_fn("cuStreamWriteValue32");
  if (fn == nullptr || addr == nullptr) return NNAB_EUNSUPPORTED;
  const CUresult r = fn((CUstream)stream, (CUdeviceptr)(uintptr_t)addr, value, 0 /* default */);
  if (r != CUDA_SUCCESS) { set_error_text("cuStreamWriteValue32 failed"); return NNAB_ECUDA; }
  return NNAB_OK;
}
int nnab_stream_wait_value32_geq(void* stream, void* addr, uint32_t value) {
  static StreamValue32Fn fn = memop_fn("cuStreamWaitValue32");
  if (fn == nullptr || addr == nullptr) return NNAB_EUNSUPPORTED;
  const CUresult r = fn((CUstream)stream, (CUdeviceptr)(uintptr_t)addr, value, 0 /* GEQ */);
  if (r != CUDA_SUCCESS) { set_error_text("cuStreamWaitValue32 failed"); return NNAB_ECUDA; }
  return NNAB_OK;
}

int nnab_block_layout_ok(int n_fft, int hop) { return tc_block_shape_ok(n_fft, hop) ? 1 : 0; }

size_t nnab_packed_block_bytes(int n_fft, int hop) { return tc_packed_block_bytes(n_fft, hop); }

int nnab_pack_basis_block(int n_fft, int hop, void* packed, void* stream) {
  if (packed == nullptr) return NNAB_EINVAL;
  return tc_pack_basis_block(n_fft, hop, packed, (cudaStream_t)stream);
}

// ------------------------------------------------------------------ STFT ----
size_t nnab_stft_workspace_bytes(int64_t B, int64_t L, int n_fft, int F, int hop, int center,
                                 int path) {
  if (!wants_tc(path, n_fft, hop)) return 0;
  const int pad = center ? n_fft / 2 : 0;
  return align_up(tc_workspace_bytes(B, L, n_fft, hop, pad), 256) +
         tc_splitk_scratch_bytes(B, F, frames_of(L, n_fft, hop, pad), n_fft);
}

int nnab_stft_forward(const float* x, int64_t B, int64_t L, int64_t x_pitch, const float* wcos,
                      const float* wsin, const void* packed, int n_fft, int F, int hop,
                      int center, int pad_mode, int out_format, float sqrt_eps, float* out,
                      int64_t T, void* workspace, size_t ws_bytes, int path, void* stream) {
  return nnab_stft_forward_ex(x, NNAB_DTYPE_F32, B, L, x_pitch, wcos, wsin, packed, n_fft, F, hop, center,
                              pad_mode, out_format, sqrt_eps, out, T, workspace, ws_bytes, path, stream);
}

static int stft_args_ok(const float* wcos, const float* wsin, int out_format) {
  if (wcos == nullptr || wsin == nullptr) return NNAB_EINVAL;
  if (out_format != NNAB_FMT_MAGNITUDE && out_format != NNAB_FMT_COMPLEX &&
      out_format != NNAB_FMT_PHASE_ANGLE)
    return NNAB_EINVAL;
  return NNAB_OK;
}

static int stft_run(const Wave& w, const float* wcos, const float* wsin, const void* packed, int n_fft, int F,
                    int hop, int out_format, float sqrt_eps, float* out, int64_t T, void* workspace,
                    size_t ws_bytes, int path, cudaStream_t stream, int* route = nullptr) {
  FramedProblem p{};
  set_wave(p, w);
  p.w_re = wcos; p.w_im = wsin; p.F = F; p.K = n_fft; p.hop = hop;
  p.scale = nullptr; p.scale_all = 1.f;
  p.fmt = out_format; p.eps = sqrt_eps; p.power = 1.f; p.out = out; p.T = T;
  p.out_bins = F; p.bin_offset = 0;
  p.route = route;
  attach_splitk_scratch(p, workspace, ws_bytes);
  return run_framed(p, packed, workspace, ws_bytes, path, stream);
}

int nnab_stft_forward_ex(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch, const float* wcos,
                         const float* wsin, const void* packed, int n_fft, int F, int hop,
                         int center, int pad_mode, int out_format, float sqrt_eps, float* out,
                         int64_t T, void* workspace, size_t ws_bytes, int path, void* stream) {
  const int pad = center ? n_fft / 2 : 0;
  int rc = check_common(x, x_dtype, B, L, x_pitch, n_fft, F, hop, pad, pad_mode, T);
  if (rc) return rc;
  if (out == nullptr || (rc = stft_args_ok(wcos, wsin, out_format))) return NNAB_EINVAL;
  if ((rc = check_arch())) return rc;
  int routes[2] = {-1, -1};  // stays -1 when nothing was enqueued
  rc = stft_run(Wave{x, x_dtype, B, L, x_pitch, pad, pad_mode, nullptr}, wcos, wsin, packed, n_fft, F, hop,
                out_format, sqrt_eps, out, T, workspace, ws_bytes, path, (cudaStream_t)stream, &routes[0]);
  if (rc == NNAB_OK) count_stft_routes(routes);
  return rc;
}

// ------------------------------------------------- Mel / Gammatone / MFCC ----
// workspace layout: [P (B,F,T) fp32][tc scratch]  (+ [mel (B,n_mels,T)][B words] for MFCC)
static size_t power_bytes(int64_t B, int F, int64_t T) {
  return align_up((size_t)B * F * T * sizeof(float), 256);
}

// table buffer: [FbEntry x F][pad to 64][int max_nnz, widest, ok, -][pad to 256][FbStep x (F + FB_STEP_PAD)]
static size_t fb_meta_offset(int F) { return align_up((size_t)F * sizeof(FbEntry), 64); }
static size_t fb_steps_offset(int F) { return align_up(fb_meta_offset(F) + 64, 256); }
size_t nnab_filterbank_table_bytes(int F) {
  return fb_steps_offset(F) + (size_t)(F + FB_STEP_PAD) * sizeof(FbStep);
}

// deterministic tile widths per table buffer (host copy of the device meta words; read at launch time):
// the one-phase kernel's nb mask and the four-phase kernel's (nb | split << 8); dense_ok: the dense kernel's
// epilogue gives every filter at most two partial sums
struct FbWidth { int nb_mask, poly_tile; bool dense_ok; };
static std::mutex g_fbw_mu;
static std::unordered_map<const void*, FbWidth> g_fb_width;
static FbWidth fb_width_of(const void* table) {
  std::lock_guard<std::mutex> lk(g_fbw_mu);
  auto it = g_fb_width.find(table);
  return it == g_fb_width.end() ? FbWidth{0, 0, false} : it->second;
}

// Replay of the dense kernel's fused-filterbank epilogue (tc_kernels.cu, FMT_FBANK) over the bin axis: each
// tc_tile_n(F) / 2 bins of an N tile run two running filter sums, and every flush is one fp32 atomic partial sum
// of that filter.  Two partial sums land on the zeroed output in either order with the same result; three do not.
static bool dense_fbank_ok(const std::vector<FbEntry>& tab, int n_fb, int F) {
  const int half = tc_tile_n(F) / 2;
  std::vector<int> sums(n_fb, 0);
  for (int f0 = 0; f0 < F; f0 += half) {
    int c0 = -1, c1 = -1;
    for (int f = f0; f < F && f < f0 + half; ++f) {
      const FbEntry& e = tab[f];
      if (e.j0 != c0) {
        if (e.j0 == c1) {
          std::swap(c0, c1);
        } else {
          if (c0 >= 0) ++sums[c0];
          c0 = e.j0;
        }
      }
      if (e.j1 != c1) {
        if (c1 >= 0) ++sums[c1];
        c1 = e.j1;
      }
    }
    if (c0 >= 0) ++sums[c0];
    if (c1 >= 0) ++sums[c1];
  }
  return std::all_of(sums.begin(), sums.end(), [](int n) { return n <= 2; });
}

int nnab_build_filterbank_table(const float* fb, int n_fb, int F, void* table, int* h_max_nnz,
                                void* stream) {
  if (fb == nullptr || table == nullptr || h_max_nnz == nullptr || n_fb <= 0 || F <= 0)
    return NNAB_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  char* base = reinterpret_cast<char*>(table);
  int* d_meta = reinterpret_cast<int*>(base + fb_meta_offset(F));
  int rc = launch_fb_table(fb, n_fb, F, reinterpret_cast<FbEntry*>(table), d_meta, s);
  if (rc) return rc;
  if (n_fb < 32768 &&
      (rc = launch_fb_steps(reinterpret_cast<const FbEntry*>(table), n_fb, F,
                            reinterpret_cast<FbStep*>(base + fb_steps_offset(F)), d_meta + 1, s)))
    return rc;
  int h_meta[4] = {0, 0, 0, 0};
  std::vector<FbEntry> h_table(F);
  NNAB_CUDA_TRY(cudaMemcpyAsync(h_meta, d_meta, sizeof(h_meta), cudaMemcpyDeviceToHost, s));
  NNAB_CUDA_TRY(cudaMemcpyAsync(h_table.data(), table, (size_t)F * sizeof(FbEntry), cudaMemcpyDeviceToHost, s));
  NNAB_CUDA_TRY(cudaStreamSynchronize(s));
  *h_max_nnz = h_meta[0];
  const bool dense_ok = dense_fbank_ok(h_table, n_fb, F);
  {
    std::lock_guard<std::mutex> lk(g_fbw_mu);
    g_fb_width[table] = (n_fb < 32768) ? FbWidth{h_meta[2], h_meta[3], dense_ok} : FbWidth{0, 0, dense_ok};
  }
  return NNAB_OK;
}

int nnab_filterbank_table_fuses(const void* table, const void* packed, int n_fft) {
  if (table == nullptr || packed == nullptr) return 0;
  if (packed_kind(packed) == PACK_BLOCK) return 1;
  // the dense kernel's fused epilogue cannot split K: a long basis takes the power spectrogram, which can
  return (fb_width_of(table).dense_ok && tc_splitk_scratch_bytes(1, 1, 1, n_fft) == 0) ? 1 : 0;
}

// ---- dense filterbank (Gammatonegram, dense mel banks) on the tensor cores -------------------------
// The block-partial STFT kernel writes |X| ** power straight into bf16 hi/lo operand planes (FMT_PLANES: one
// row per frame, 4 B per value, no fp32 (B, F, T) intermediate), a second tensor-core launch contracts the rows
// with the re-indexed bank (real GEMM on the complex kernel, FMT_REALPAIR) and writes (B, n_fb, T).
// Workspace: [signal planes of the STFT][operand planes][bank fp32 re | im][packed bank].
static bool fb_planes_enabled() {
  if (const char* e = getenv("NNAB_FB_PLANES")) return atoi(e) != 0;
  // on by default (tests/test_zz_gpu_fb_planes.py: oracle parity, bit-repeatable); 0 = fp32 (B, F, T) power
  // spectrogram + CUDA-core filterbank GEMM
  return true;
}

struct FbPlanes {
  int nb, n_tiles, phases, kp, fh;
  int64_t rows;  // B * T frame rows
  size_t off_planes, off_w, off_packed, total;
};

static bool fb_planes_layout(int64_t B, int64_t L, int n_fft, int F, int hop, int pad, int64_t T, int n_fb,
                             FbPlanes* o) {
  if (!tc_block_shape_ok(n_fft, hop) || F != n_fft / 2 + 1 || n_fb < 1 || T <= 0 || B <= 0) return false;
  tc_block_tile_geometry(n_fft, hop, &o->nb, &o->n_tiles, &o->phases);
  o->kp = (o->nb * o->n_tiles * o->phases + 63) / 64 * 64;
  o->fh = (n_fb + 1) / 2;
  o->rows = B * T;
  if (o->rows >= (1ll << 31) || o->kp > 32768) return false;
  size_t off = align_up(tc_workspace_bytes(B, L, n_fft, hop, pad), 256);
  o->off_planes = off; off += align_up((size_t)2 * o->rows * o->kp * 2, 256);
  o->off_w = off;      off += 2 * align_up((size_t)o->fh * o->kp * sizeof(float), 256);
  o->off_packed = off; off += align_up(tc_packed_bytes(o->fh, o->kp), 256);
  o->total = off + 256;
  return true;
}

static bool fused_fbank(int path, const void* packed, const void* fb_table, int n_fft, int hop) {
  return fb_table != nullptr && packed != nullptr && path != NNAB_PATH_SIMT &&
         wants_tc(path, n_fft, hop);
}

static size_t filterbank_ws_bytes(int64_t B, int64_t L, int n_fft, int F, int hop, int pad, int n_fb, int path,
                                  int has_table) {
  const int64_t T = frames_of(L, n_fft, hop, pad);
  const bool tc = wants_tc(path, n_fft, hop);
  size_t n = 0;
  if (has_table && tc) {
    n += tc_workspace_bytes(B, L, n_fft, hop, pad);
  } else {  // un-fused: (B,F,T) power spectrogram, then the contraction's planes and a long basis's split-K scratch
    n += power_bytes(B, F, T);
    if (tc) n += align_up(tc_workspace_bytes(B, L, n_fft, hop, pad), 256) + tc_splitk_scratch_bytes(B, F, T, n_fft);
  }
  if (!has_table && tc) {  // dense bank on the tensor cores: operand planes instead of the fp32 spectrogram
    FbPlanes fp;
    if (fb_planes_layout(B, L, n_fft, F, hop, pad, T, n_fb, &fp) && fp.total > n) n = fp.total;
  }
  return n;
}

size_t nnab_filterbank_workspace_bytes(int64_t B, int64_t L, int n_fft, int F, int hop,
                                       int center, int n_fb, int path, int has_table) {
  return filterbank_ws_bytes(B, L, n_fft, F, hop, center ? n_fft / 2 : 0, n_fb, path, has_table);
}

static int power_spectrogram(const Wave& w, const float* wcos, const float* wsin, const void* packed,
                             int n_fft, int F, int hop, float sqrt_eps,
                             float power, float* P, int64_t T, void* tc_ws, size_t tc_ws_bytes,
                             int path, cudaStream_t stream, int* route) {
  FramedProblem p{};
  set_wave(p, w);
  p.w_re = wcos; p.w_im = wsin; p.F = F; p.K = n_fft; p.hop = hop;
  p.scale = nullptr; p.scale_all = 1.f;
  p.fmt = FMT_POWER; p.eps = sqrt_eps; p.power = power; p.out = P; p.T = T;
  p.out_bins = F; p.bin_offset = 0;
  p.route = route;
  attach_splitk_scratch(p, tc_ws, tc_ws_bytes);
  return run_framed(p, packed, tc_ws, tc_ws_bytes, path, stream);
}

int nnab_stft_filterbank_forward(const float* x, int64_t B, int64_t L, int64_t x_pitch,
                                 const float* wcos, const float* wsin, const void* packed,
                                 int n_fft, int F, int hop, int center, int pad_mode,
                                 float sqrt_eps, float power, const float* fb, int n_fb,
                                 const void* fb_table, float* out, int64_t T, void* workspace,
                                 size_t ws_bytes, int path, void* stream) {
  return nnab_stft_filterbank_forward_ex(x, NNAB_DTYPE_F32, B, L, x_pitch, wcos, wsin, packed, n_fft, F, hop,
                                         center, pad_mode, sqrt_eps, power, fb, n_fb, fb_table, out, T,
                                         workspace, ws_bytes, path, stream);
}

static int filterbank_args_ok(const float* wcos, const float* wsin, const float* fb, int n_fb) {
  return (wcos == nullptr || wsin == nullptr || fb == nullptr || n_fb <= 0) ? NNAB_EINVAL : NNAB_OK;
}

static int filterbank_run(const Wave& w, const float* wcos, const float* wsin, const void* packed, int n_fft,
                          int F, int hop, float sqrt_eps, float power, const float* fb, int n_fb,
                          const void* fb_table, float* out, int64_t T, void* workspace, size_t ws_bytes, int path,
                          cudaStream_t s, int (*routes)[2] = nullptr) {
  const int64_t B = w.B, L = w.L;
  const int pad = w.pad;
  int rc;
  int scratch[2];
  int (&r)[2] = routes != nullptr ? *routes : scratch;
  // the fused epilogue on a dense basis only when its atomics stay order-independent (nnab_filterbank_table_fuses)
  if (fused_fbank(path, packed, fb_table, n_fft, hop) && nnab_filterbank_table_fuses(fb_table, packed, n_fft)) {
    FramedProblem p{};
    set_wave(p, w);
    p.w_re = wcos; p.w_im = wsin; p.F = F; p.K = n_fft; p.hop = hop;
    p.scale = nullptr; p.scale_all = 1.f;
    p.fmt = FMT_FBANK; p.eps = sqrt_eps; p.power = power; p.out = out; p.T = T;
    p.out_bins = n_fb; p.bin_offset = 0;
    p.fb_table = reinterpret_cast<const FbEntry*>(fb_table); p.n_fb = n_fb;
    p.fb_steps = reinterpret_cast<const FbStep*>(reinterpret_cast<const char*>(fb_table) + fb_steps_offset(F));
    const FbWidth fw = fb_width_of(fb_table);
    p.fb_nb_mask = fw.nb_mask;
    p.fb_poly_tile = fw.poly_tile;
    p.route = &r[0];
    if (tc_supported(p, packed)) {
      const size_t need = tc_workspace_bytes(B, L, n_fft, hop, pad);
      if (workspace == nullptr || ws_bytes < need) return NNAB_EWORKSPACE;
      // the epilogue accumulates filter sums with fp32 atomics: start from zero
      NNAB_CUDA_TRY(cudaMemsetAsync(out, 0, (size_t)B * n_fb * T * sizeof(float), s));
      if ((rc = run_framed(p, packed, workspace, ws_bytes, NNAB_PATH_TCGEN05, s))) return rc;
      r[1] = NNAB_STFT_FB_FUSED;
      return NNAB_OK;
    }
  }
  const size_t need = filterbank_ws_bytes(B, L, n_fft, F, hop, pad, n_fb, path, 0);
  if (workspace == nullptr || ws_bytes < need) return NNAB_EWORKSPACE;
  FbPlanes fp;
  if (fb_planes_enabled() && path != NNAB_PATH_SIMT && packed != nullptr && packed_kind(packed) == PACK_BLOCK &&
      wants_tc(path, n_fft, hop) && B <= 65535 &&
      fb_planes_layout(B, L, n_fft, F, hop, pad, T, n_fb, &fp) && ws_bytes >= fp.total) {
    char* ws = reinterpret_cast<char*>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    __nv_bfloat16* planes = reinterpret_cast<__nv_bfloat16*>(ws + fp.off_planes);
    float* w_re = reinterpret_cast<float*>(ws + fp.off_w);
    float* w_im = reinterpret_cast<float*>(ws + fp.off_w + align_up((size_t)fp.fh * fp.kp * sizeof(float), 256));
    void* bank = ws + fp.off_packed;
    const int64_t plane_stride = fp.rows * fp.kp;
    // 1. STFT -> |X| ** power as operand planes (block-partial kernel, FMT_PLANES)
    FramedProblem p{};
    set_wave(p, w);
    p.w_re = wcos; p.w_im = wsin; p.F = F; p.K = n_fft; p.hop = hop;
    p.scale = nullptr; p.scale_all = 1.f;
    p.fmt = FMT_PLANES; p.eps = sqrt_eps; p.power = power; p.out = reinterpret_cast<float*>(planes); p.T = T;
    p.out_bins = F; p.bin_offset = 0;
    p.planes_stride = plane_stride; p.planes_pitch = fp.kp;
    p.route = &r[0];
    // 2. rows x bank on the dense kernel: every frame is one "hop" of kp samples
    FramedProblem g{};
    g.x = nullptr; g.B = B; g.L = T * fp.kp; g.x_pitch = T * fp.kp;
    g.w_re = w_re; g.w_im = w_im; g.F = fp.fh; g.K = fp.kp; g.hop = fp.kp;
    g.pad = 0; g.pad_mode = NNAB_PAD_CONSTANT; g.scale = nullptr; g.scale_all = 1.f;
    g.fmt = FMT_REALPAIR; g.eps = 0.f; g.power = 1.f; g.out = out; g.T = T;
    g.out_bins = n_fb; g.bin_offset = 0;
    g.presplit = planes; g.presplit_t_slots = T; g.presplit_plane_stride = plane_stride;
    // a shape either contraction rejects takes the fp32 path below, before anything is enqueued
    if (tc_supported(p, packed) && tc_supported(g)) {
      // the re-indexed bank (tiny: fh x kp) and its bf16 hi/lo packing
      if ((rc = launch_fb_tile_bank(fb, n_fb, F, fp.nb, fp.n_tiles, fp.phases, fp.kp, fp.fh, w_re, w_im, s)))
        return rc;
      if ((rc = tc_pack_basis(w_re, w_im, fp.fh, fp.kp, bank, s))) return rc;
      // columns no tile writes (kp is the 64-multiple above n_tiles * phases * nb): finite zeros in both planes
      const int written = fp.nb * fp.n_tiles * fp.phases;
      if (fp.kp > written)
        NNAB_CUDA_TRY(cudaMemset2DAsync(planes + written, (size_t)fp.kp * 2, 0, (size_t)(fp.kp - written) * 2,
                                        (size_t)(2 * fp.rows), s));
      if ((rc = run_framed(p, packed, ws, fp.off_planes, NNAB_PATH_TCGEN05, s))) return rc;
      if ((rc = run_framed(g, bank, nullptr, 0, NNAB_PATH_TCGEN05, s))) return rc;
      r[1] = NNAB_STFT_FB_PLANES;
      return NNAB_OK;
    }
  }
  float* P = (float*)workspace;
  const size_t pb = power_bytes(B, F, T);
  rc = power_spectrogram(w, wcos, wsin, packed, n_fft, F, hop, sqrt_eps, power, P, T, (char*)workspace + pb,
                         ws_bytes - pb, path, s, &r[0]);
  if (rc || (rc = launch_filterbank(P, fb, B, F, T, n_fb, out, s))) return rc;
  r[1] = NNAB_STFT_FB_GEMM;
  return NNAB_OK;
}

int nnab_stft_filterbank_forward_ex(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch,
                                    const float* wcos, const float* wsin, const void* packed,
                                    int n_fft, int F, int hop, int center, int pad_mode,
                                    float sqrt_eps, float power, const float* fb, int n_fb,
                                    const void* fb_table, float* out, int64_t T, void* workspace,
                                    size_t ws_bytes, int path, void* stream) {
  const int pad = center ? n_fft / 2 : 0;
  int rc = check_common(x, x_dtype, B, L, x_pitch, n_fft, F, hop, pad, pad_mode, T);
  if (rc) return rc;
  if (out == nullptr || filterbank_args_ok(wcos, wsin, fb, n_fb)) return NNAB_EINVAL;
  if ((rc = check_arch())) return rc;
  int routes[2] = {-1, -1};
  rc = filterbank_run(Wave{x, x_dtype, B, L, x_pitch, pad, pad_mode, nullptr}, wcos, wsin, packed, n_fft, F, hop,
                      sqrt_eps, power, fb, n_fb, fb_table, out, T, workspace, ws_bytes, path, (cudaStream_t)stream,
                      &routes);
  if (rc == NNAB_OK) count_stft_routes(routes);
  return rc;
}

static size_t mel_bytes(int64_t B, int n_mels, int64_t T) {
  return align_up((size_t)B * n_mels * T * sizeof(float), 256);
}

static size_t mfcc_ws_bytes(int64_t B, int64_t L, int n_fft, int F, int hop, int pad, int n_mels, int path) {
  const int64_t T = frames_of(L, n_fft, hop, pad);
  // the un-fused size is the upper bound (a huge batch can still fall back to it)
  const size_t fbw = filterbank_ws_bytes(B, L, n_fft, F, hop, pad, n_mels, path, 0);
  return align_up(fbw, 256) + mel_bytes(B, n_mels, T) + align_up((size_t)B * sizeof(unsigned int), 256);
}

size_t nnab_mfcc_workspace_bytes(int64_t B, int64_t L, int n_fft, int F, int hop, int center,
                                 int n_mels, int path, int has_table) {
  (void)has_table;
  return mfcc_ws_bytes(B, L, n_fft, F, hop, center ? n_fft / 2 : 0, n_mels, path);
}

int nnab_mfcc_forward(const float* x, int64_t B, int64_t L, int64_t x_pitch, const float* wcos,
                      const float* wsin, const void* packed, int n_fft, int F, int hop,
                      int center, int pad_mode, float sqrt_eps, float power,
                      const float* mel_basis, int n_mels, const void* fb_table, float amin,
                      float ref, float top_db, const float* dct, int n_mfcc, float* out,
                      int64_t T, void* workspace, size_t ws_bytes, int path, void* stream) {
  return nnab_mfcc_forward_ex(x, NNAB_DTYPE_F32, B, L, x_pitch, wcos, wsin, packed, n_fft, F, hop, center,
                              pad_mode, sqrt_eps, power, mel_basis, n_mels, fb_table, amin, ref, top_db, dct,
                              n_mfcc, out, T, workspace, ws_bytes, path, stream);
}

static int mfcc_args_ok(const float* wcos, const float* wsin, const float* mel_basis, int n_mels,
                        const float* dct, int n_mfcc, float amin) {
  if (wcos == nullptr || wsin == nullptr || mel_basis == nullptr || dct == nullptr || n_mels <= 0 ||
      n_mfcc <= 0 || !(amin > 0.f))
    return NNAB_EINVAL;
  return NNAB_OK;
}

static int mfcc_run(const Wave& w, const float* wcos, const float* wsin, const void* packed, int n_fft, int F,
                    int hop, float sqrt_eps, float power, const float* mel_basis, int n_mels,
                    const void* fb_table, float amin, float ref, float top_db, const float* dct, int n_mfcc,
                    float* out, int64_t T, void* workspace, size_t ws_bytes, int path, cudaStream_t stream,
                    int (*routes)[2] = nullptr) {
  const size_t need = mfcc_ws_bytes(w.B, w.L, n_fft, F, hop, w.pad, n_mels, path);
  if (workspace == nullptr || ws_bytes < need) return NNAB_EWORKSPACE;
  if (w.B > MFCC_MAX_CLIPS) return NNAB_EUNSUPPORTED;  // refused before the mel stage is enqueued
  const size_t fbw = align_up(filterbank_ws_bytes(w.B, w.L, n_fft, F, hop, w.pad, n_mels, path, 0), 256);
  float* mel = (float*)((char*)workspace + fbw);
  unsigned int* scratch = (unsigned int*)((char*)workspace + fbw + mel_bytes(w.B, n_mels, T));
  int rc = filterbank_run(w, wcos, wsin, packed, n_fft, F, hop, sqrt_eps, power, mel_basis, n_mels, fb_table,
                          mel, T, workspace, fbw, path, stream, routes);
  if (rc) return rc;
  return launch_mfcc_tail(mel, w.B, n_mels, T, amin, ref, top_db, dct, n_mfcc, out, scratch, stream);
}

int nnab_mfcc_forward_ex(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch, const float* wcos,
                         const float* wsin, const void* packed, int n_fft, int F, int hop,
                         int center, int pad_mode, float sqrt_eps, float power,
                         const float* mel_basis, int n_mels, const void* fb_table, float amin,
                         float ref, float top_db, const float* dct, int n_mfcc, float* out,
                         int64_t T, void* workspace, size_t ws_bytes, int path, void* stream) {
  const int pad = center ? n_fft / 2 : 0;
  int rc = check_common(x, x_dtype, B, L, x_pitch, n_fft, F, hop, pad, pad_mode, T);
  if (rc) return rc;
  if (out == nullptr || mfcc_args_ok(wcos, wsin, mel_basis, n_mels, dct, n_mfcc, amin)) return NNAB_EINVAL;
  if ((rc = check_arch())) return rc;
  int routes[2] = {-1, -1};
  rc = mfcc_run(Wave{x, x_dtype, B, L, x_pitch, pad, pad_mode, nullptr}, wcos, wsin, packed, n_fft, F, hop,
                sqrt_eps, power, mel_basis, n_mels, fb_table, amin, ref, top_db, dct, n_mfcc, out, T, workspace,
                ws_bytes, path, (cudaStream_t)stream, &routes);
  if (rc == NNAB_OK) count_stft_routes(routes);
  return rc;
}

// ------------------------------------------------------------- CQT1992v2 ----
size_t nnab_cqt1992v2_workspace_bytes(int64_t B, int64_t L, int width, int n_bins, int hop,
                                      int center, int path) {
  if (!wants_tc(path, width, hop)) return 0;
  const int pad = center ? width / 2 : 0;
  return align_up(tc_workspace_bytes(B, L, width, hop, pad), 256) +
         tc_splitk_scratch_bytes(B, n_bins, frames_of(L, width, hop, pad), width);
}

static int cqt1992v2_args_ok(const float* k_real, const float* k_imag, int out_format) {
  if (k_real == nullptr || k_imag == nullptr) return NNAB_EINVAL;
  if (out_format != NNAB_FMT_MAGNITUDE && out_format != NNAB_FMT_COMPLEX &&
      out_format != NNAB_FMT_PHASE_UNIT)
    return NNAB_EINVAL;
  return NNAB_OK;
}

static int cqt1992v2_run(const Wave& w, const float* k_real, const float* k_imag, const void* packed,
                         const int32_t* h_k_begin, const int32_t* h_k_end, int n_bins, int width, int hop,
                         const float* scale, float scale_all, int out_format, float sqrt_eps, float* out,
                         int64_t T, void* workspace, size_t ws_bytes, int path, cudaStream_t stream,
                         int* route = nullptr) {
  FramedProblem p{};
  set_wave(p, w);
  p.w_re = k_real; p.w_im = k_imag; p.F = n_bins; p.K = width; p.hop = hop;
  p.scale = scale; p.scale_all = scale_all;
  p.fmt = out_format; p.eps = sqrt_eps; p.power = 1.f; p.out = out; p.T = T;
  p.out_bins = n_bins; p.bin_offset = 0;
  p.h_k_begin = h_k_begin; p.h_k_end = h_k_end;
  p.route = route;
  attach_splitk_scratch(p, workspace, ws_bytes);
  return run_framed(p, packed, workspace, ws_bytes, path, stream);
}

int nnab_cqt1992v2_forward(const float* x, int64_t B, int64_t L, int64_t x_pitch,
                           const float* k_real, const float* k_imag, const void* packed,
                           const int32_t* h_k_begin, const int32_t* h_k_end, int n_bins,
                           int width, int hop, int center, int pad_mode, const float* scale,
                           float scale_all, int out_format, float sqrt_eps, float* out,
                           int64_t T, void* workspace, size_t ws_bytes, int path,
                           void* stream) {
  return nnab_cqt1992v2_forward_ex(x, NNAB_DTYPE_F32, B, L, x_pitch, k_real, k_imag, packed, h_k_begin,
                                   h_k_end, n_bins, width, hop, center, pad_mode, scale, scale_all, out_format,
                                   sqrt_eps, out, T, workspace, ws_bytes, path, stream);
}

int nnab_cqt1992v2_forward_ex(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch,
                              const float* k_real, const float* k_imag, const void* packed,
                              const int32_t* h_k_begin, const int32_t* h_k_end, int n_bins,
                              int width, int hop, int center, int pad_mode, const float* scale,
                              float scale_all, int out_format, float sqrt_eps, float* out,
                              int64_t T, void* workspace, size_t ws_bytes, int path,
                              void* stream) {
  const int pad = center ? width / 2 : 0;
  int rc = check_common(x, x_dtype, B, L, x_pitch, width, n_bins, hop, pad, pad_mode, T);
  if (rc) return rc;
  if (out == nullptr || cqt1992v2_args_ok(k_real, k_imag, out_format)) return NNAB_EINVAL;
  if ((rc = check_arch())) return rc;
  int route = -1;  // stays -1 when nothing was enqueued
  rc = cqt1992v2_run(Wave{x, x_dtype, B, L, x_pitch, pad, pad_mode, nullptr}, k_real, k_imag, packed, h_k_begin,
                     h_k_end, n_bins, width, hop, scale, scale_all, out_format, sqrt_eps, out, T, workspace,
                     ws_bytes, path, (cudaStream_t)stream, &route);
  if (rc == NNAB_OK) count_cq1992_route(route, g_cq1992_routes);
  return rc;
}

// ------------------------------------------------ CQT2010v2 / VQT pyramid ----
// (level lengths: decimated_len, common.cuh)
static size_t pyramid_level_bytes(int64_t B, int64_t L, int early_factor) {
  // [early (B, L0)] + ping/pong level buffers (B, <= L0/2 + 1)
  const int64_t L0 = early_factor > 1 ? decimated_len(L, early_factor) : L;
  size_t n = 0;
  if (early_factor > 1) n += align_up((size_t)B * align_up((size_t)L0, 4) * sizeof(float), 256);
  const size_t half = align_up((size_t)(L0 / 2 + 1), 4);
  n += 2 * align_up((size_t)B * half * sizeof(float), 256);
  return n;
}

// ---- plan of the all-tensor-core pyramid -----------------------------------------
constexpr int FIR_TAPS = 256;
constexpr int FIR_OFF = 128;  // sample m of a level sits at plane offset 128 + m in FIR inputs

struct PyrLevel {
  int64_t len;
  int hop, width, pad, mode;
  bool presplit;          // octave reads pre-split planes (single frame phase)
  size_t pc, pf, y32;     // workspace offsets (SIZE_MAX = not needed)
  int64_t pc_pitch, pc_plane, pf_pitch, pf_plane, y32_pitch;
};

static size_t planes_bytes(int64_t B, int64_t L, int K, int hop, int pad, int64_t* pitch,
                           int64_t* plane) {
  int64_t t_slots = 0, ps = 0;
  int he = 0;
  tc_split_geometry(B, L, K, hop, pad, &t_slots, &ps, &he);
  if (pitch) *pitch = t_slots * he;
  if (plane) *plane = ps;
  return align_up((size_t)(2 * ps) * 2, 256);
}

// Fills lv[0..n_octaves) and returns the workspace size; `pf_early` receives the offset of
// the raw-signal FIR input when early downsampling is active, `scratch` the offset of the
// split-signal scratch of the octaves that run from fp32.
static size_t plan_pyramid(int64_t B, int64_t L, int n_octaves, int early_factor, int hop,
                           const int32_t* widths, int fixed_width, int pad_mode, PyrLevel* lv,
                           size_t* pf_early, size_t* scratch) {
  size_t off = 0;
  auto take = [&](size_t n) { size_t o = off; off += n; return o; };
  int64_t len = L;
  if (early_factor > 1) {
    *pf_early = take(planes_bytes(B, L, tc_fir_k(FIR_TAPS, early_factor), 128 * early_factor,
                                  FIR_OFF, nullptr, nullptr));
    len = decimated_len(L, early_factor);
  }
  int cur_hop = hop;
  for (int i = 0; i < n_octaves; ++i) {
    if (i > 0) { len = decimated_len(len, 2); cur_hop /= 2; }
    PyrLevel& l = lv[i];
    l.len = len; l.hop = cur_hop;
    l.width = widths ? widths[i] : fixed_width;
    l.pad = l.width / 2;
    l.mode = (pad_mode == NNAB_PAD_REFLECT && l.pad >= len) ? NNAB_PAD_CONSTANT : pad_mode;
    l.presplit = cur_hop > 0 && (cur_hop % 8) == 0;
    l.pc = l.pf = l.y32 = SIZE_MAX;
    l.pc_pitch = l.pc_plane = l.pf_pitch = l.pf_plane = l.y32_pitch = 0;
    if (len <= 0 || cur_hop <= 0) continue;
    const bool from_x = (i == 0 && early_factor <= 1);  // level 0 is the caller's fp32 input
    if (l.presplit)
      l.pc = take(planes_bytes(B, len, l.width, cur_hop, l.pad, &l.pc_pitch, &l.pc_plane));
    else if (!from_x) {
      l.y32_pitch = (int64_t)align_up((size_t)len, 8);
      l.y32 = take(align_up((size_t)B * l.y32_pitch * sizeof(float), 256));
    }
    if (i < n_octaves - 1)
      l.pf = take(planes_bytes(B, len, tc_fir_k(FIR_TAPS, 2), 256, FIR_OFF, &l.pf_pitch,
                               &l.pf_plane));
  }
  // scratch for octaves that run from fp32 (several frame phases): sized for the first such level
  *scratch = off;
  for (int i = 0; i < n_octaves; ++i)
    if (!lv[i].presplit && lv[i].len > 0 && lv[i].hop > 0) {
      off += tc_workspace_bytes(B, lv[i].len, lv[i].width, lv[i].hop, lv[i].pad);
      break;
    }
  return off;
}

// ---------------------------------------------------------------------------------------------
// Pyramid, second generation (round 2): ONE plane set per level, shared by the level's octave CQT
// (reflect margins of `pad` samples, frames every `hop`) and by the FIR stage that produces the next
// level (256-sample rows, banded taps, clip edges recomputed: launch_fir_stage_tc).  Per level and
// sample: one 4-byte write and one read by each consumer, instead of two differently padded copies.
// ---------------------------------------------------------------------------------------------
struct Lvl2 {
  int64_t len;
  int hop, width, pad, mode;
  bool presplit;        // the octave CQT reads the planes directly (single frame phase)
  bool planes;          // the level has planes (CQT and / or FIR source)
  size_t pc, y32;       // workspace offsets (SIZE_MAX = none)
  int64_t pitch, plane, t_slots, y32_pitch;
};

static int64_t gcd64(int64_t a, int64_t b) { return b == 0 ? a : gcd64(b, a % b); }

// false: the shape does not fit this plan.  `scratch` receives the offset of the split-signal
// scratch of the octaves that run from fp32, `total` the workspace size.
static bool plan_pyramid2(int64_t B, int64_t L, int n_octaves, int hop, const int32_t* widths,
                          int fixed_width, int pad_mode, Lvl2* lv, size_t* scratch, size_t* total) {
  size_t off = 0;
  auto take = [&](size_t n) { size_t o = off; off += align_up(n, 256); return o; };
  int64_t len = L;
  int cur_hop = hop;
  for (int i = 0; i < n_octaves; ++i) {
    if (i > 0) { len = decimated_len(len, 2); cur_hop /= 2; }
    Lvl2& l = lv[i];
    l.len = len; l.hop = cur_hop;
    l.width = widths ? widths[i] : fixed_width;
    l.pad = l.width / 2;
    if (len <= 0 || cur_hop <= 0) return false;
    l.mode = (pad_mode == NNAB_PAD_REFLECT && l.pad >= len) ? NNAB_PAD_CONSTANT : pad_mode;
    l.presplit = (cur_hop % 8) == 0;
    const bool fir_src = i < n_octaves - 1;
    l.planes = l.presplit || fir_src;
    l.pc = l.y32 = SIZE_MAX;
    l.pitch = l.plane = l.t_slots = l.y32_pitch = 0;
    if (fir_src && l.pad != 128) return false;  // FIR frame origin = CQT padding origin (256-tap banks)
    if (l.planes) {
      const int he = l.presplit ? cur_hop : 8;  // planes of multi-phase levels only feed the FIR
      const int kpad = (l.width + 63) / 64 * 64;
      int64_t need = len + 2 * (int64_t)l.pad + kpad;
      if (fir_src) {
        const int64_t FT = (decimated_len(len, 2) + 127) / 128;
        const int64_t rows = FT + 2;
        if (256 * rows > need) need = 256 * rows;
      }
      const int64_t gran = (int64_t)he / gcd64(he, 256) * 256;  // lcm(he, 256)
      l.pitch = (need + gran - 1) / gran * gran;
      l.t_slots = l.pitch / he;
      const int64_t rows = B * l.t_slots + (kpad + he - 1) / he + 1;
      l.plane = (rows * he + 255) / 256 * 256;
      l.pc = take((size_t)2 * l.plane * 2);
    }
    if (!l.presplit && i > 0) {
      l.y32_pitch = (int64_t)align_up((size_t)len, 8);
      l.y32 = take((size_t)B * l.y32_pitch * sizeof(float));
    }
  }
  // scratch for octaves that run from fp32 (several frame phases): sized for the first such level
  *scratch = off;
  for (int i = 0; i < n_octaves; ++i)
    if (!lv[i].presplit) {
      off += tc_workspace_bytes(B, lv[i].len, lv[i].width, lv[i].hop, lv[i].pad) + 256;
      break;
    }
  *total = off;
  return true;
}

size_t nnab_packed_fir_bytes(int taps, int dec) { return tc_packed_fir_bytes(taps, dec); }
int nnab_pack_fir(const float* fir, int taps, int dec, void* packed, void* stream) {
  if (fir == nullptr || packed == nullptr || taps <= 0 || dec < 1) return NNAB_EINVAL;
  return tc_pack_fir(fir, taps, dec, packed, (cudaStream_t)stream);
}

int nnab_debug_varn_plan(const int32_t* h_k_begin, const int32_t* h_k_end, int n_bins, int width,
                         int want_chunks, int32_t* order, int32_t* groups, int32_t* chunk_begin,
                         int32_t* n_blocks, int32_t* n_chunks) {
  if (order == nullptr || groups == nullptr || chunk_begin == nullptr || n_blocks == nullptr ||
      n_chunks == nullptr || n_bins <= 0 || width <= 0)
    return NNAB_EINVAL;
  return tc_varn_plan_export(h_k_begin, h_k_end, n_bins, width, want_chunks, order, groups,
                             chunk_begin, n_blocks, n_chunks);
}

int nnab_debug_ola_plan(int F_out, int K_gemm, int64_t M_rows, int k_splits_hint, double* out) {
  if (out == nullptr || F_out <= 0 || K_gemm <= 0 || M_rows < 0) return NNAB_EINVAL;
  const OlaPlan o = tc_ola_plan(F_out, K_gemm, M_rows, k_splits_hint);
  out[0] = o.supported;
  out[1] = o.bn;
  out[2] = o.n_tiles;
  out[3] = o.k_splits;
  out[4] = o.exec_flops;
  return NNAB_OK;
}

int nnab_fir_decimate(const float* x, int64_t B, int64_t L, int64_t x_pitch, const float* fir,
                      int taps, int factor, float* y, int64_t Ly, void* stream) {
  if (x == nullptr || fir == nullptr || y == nullptr || B < 0 || L <= 0 || x_pitch < L || taps <= 0 ||
      factor < 1)
    return NNAB_EINVAL;
  const int half = (taps - 1) / 2;
  if (L + 2 * (int64_t)half < taps || Ly != (L + 2 * (int64_t)half - taps) / factor + 1)
    return NNAB_EINVAL;
  int rc = check_arch();
  if (rc) return rc;
  return launch_fir_decimate(x, B, L, x_pitch, fir, taps, factor, y, Ly, Ly, (cudaStream_t)stream);
}

int nnab_fir_decimate_adjoint(const float* g, int64_t B, int64_t Ly, int64_t g_pitch,
                              const float* fir, int taps, int factor, float* dx, int64_t L,
                              void* stream) {
  if (g == nullptr || fir == nullptr || dx == nullptr || B < 0 || L <= 0 || Ly <= 0 || g_pitch < Ly ||
      taps <= 0 || factor < 1)
    return NNAB_EINVAL;
  const int half = (taps - 1) / 2;
  if (L + 2 * (int64_t)half < taps || Ly != (L + 2 * (int64_t)half - taps) / factor + 1)
    return NNAB_EINVAL;
  int rc = check_arch();
  if (rc) return rc;
  return launch_fir_decimate_adjoint(g, B, Ly, g_pitch, fir, taps, factor, dx, L, L,
                                     (cudaStream_t)stream);
}

size_t nnab_cqt_pyramid_workspace_bytes(int64_t B, int64_t L, int n_octaves, int early_factor,
                                        int max_width, int hop, int path) {
  size_t n = pyramid_level_bytes(B, L, early_factor);
  if (path != NNAB_PATH_SIMT) {
    // (a) per-octave tensor-core path: split-signal scratch of the largest level
    const int64_t L0 = early_factor > 1 ? decimated_len(L, early_factor) : L;
    n += tc_workspace_bytes(B, L0, max_width, hop, max_width / 2);
    // (b) all-tensor-core pyramid: every level's planes (upper bound with max_width)
    if (n_octaves <= 32) {
      PyrLevel lv[32];
      size_t pf_early = 0, scratch = 0;
      const size_t full = plan_pyramid(B, L, n_octaves, early_factor, hop, nullptr, max_width,
                                       NNAB_PAD_REFLECT, lv, &pf_early, &scratch) + 1024;
      if (full > n) n = full;
      Lvl2 lv2[32];
      size_t full2 = 0;
      if (early_factor <= 1 && plan_pyramid2(B, L, n_octaves, hop, nullptr, max_width, NNAB_PAD_REFLECT,
                                             lv2, &scratch, &full2)) {
        full2 += 2048;
        if (full2 > n) n = full2;
      }
    }
  }
  return n;
}

// Arguments of one nnab_cqt_pyramid_forward call, shared by its three plans (same order as the call's).
struct PyramidCall {
  const void* x; int x_dtype; int64_t B, L, x_pitch; int n_octaves;
  const float* const* k_real; const float* const* k_imag; const void* const* packed; const int32_t* widths;
  int n_filters; const float* lowpass; const void* lowpass_packed; const void* early_packed;
  int early_factor, hop, pad_mode, n_bins; const float* scale; float scale_all; int out_format; float sqrt_eps;
  float* out; int64_t T;
  char* ws;  // the workspace aligned up to 256 bytes (the plans' size checks leave room for it)
  size_t ws_bytes; cudaStream_t s;
};

// Octave i (0 = top) on a level of `len` samples framed every `hop`: its n_filters bins land
// n_filters * (i + 1) rows below the top of the output, and the per-bin scale, indexed by output
// row, is shifted by the same offset.
static FramedProblem octave_problem(const PyramidCall& c, int i, int64_t len, int hop, int pad_mode) {
  FramedProblem p{};
  p.B = c.B; p.L = len;
  p.w_re = c.k_real[i]; p.w_im = c.k_imag[i]; p.F = c.n_filters; p.K = c.widths[i]; p.hop = hop;
  p.pad = p.K / 2; p.pad_mode = pad_mode; p.scale_all = c.scale_all;
  p.fmt = c.out_format; p.eps = c.sqrt_eps; p.power = 1.f; p.out = c.out; p.T = c.T;
  p.out_bins = c.n_bins;
  p.bin_offset = c.n_bins - c.n_filters * (i + 1);
  p.scale = c.scale ? c.scale + p.bin_offset : nullptr;
  return p;
}

// Octave i of the gen-2 plan: on the level planes (one frame phase) or on the fp32 level.
static FramedProblem octave2_problem(const PyramidCall& c, const Lvl2& l, int i) {
  FramedProblem p = octave_problem(c, i, l.len, l.hop, l.mode);
  if (l.presplit) {
    p.presplit = c.ws + l.pc;
    p.presplit_t_slots = l.t_slots;
    p.presplit_plane_stride = l.plane;
  } else if (i == 0) {  // the caller's waveform
    p.x = c.x; p.x_dtype = c.x_dtype; p.x_pitch = c.x_pitch;
  } else {
    p.x = c.ws + l.y32; p.x_pitch = l.y32_pitch;
  }
  return p;
}

// Gen-2 plan of a call: NNAB_OK with lv and the scratch offset filled, NNAB_EUNSUPPORTED when the
// call needs another plan, NNAB_EINVAL when an octave's frame count is not T.
static int select_fused2(const PyramidCall& c, Lvl2* lv, size_t* scratch) {
  if (c.n_octaves > 32 || c.B > 65535) return NNAB_EUNSUPPORTED;
  size_t need = 0;
  if (!plan_pyramid2(c.B, c.L, c.n_octaves, c.hop, c.widths, 0, c.pad_mode, lv, scratch, &need))
    return NNAB_EUNSUPPORTED;
  if (need + 512 > c.ws_bytes) return NNAB_EUNSUPPORTED;
  for (int i = 0; i < c.n_octaves; ++i)
    if (frames_of(lv[i].len, lv[i].width, lv[i].hop, lv[i].pad) != c.T) return NNAB_EINVAL;
  // an octave the octave kernel does not take runs on the dense kernel (the FIR stages fit by construction)
  for (int i = 0; i < c.n_octaves; ++i) {
    const FramedProblem p = octave2_problem(c, lv[i], i);
    if (!octave_tc_ok(p) && !tc_supported(p)) return NNAB_EUNSUPPORTED;
  }
  return NNAB_OK;
}

static int pyramid_fused2(const PyramidCall& c, const Lvl2* lv, size_t scratch_off) {
  const int64_t B = c.B;
  char* const ws = c.ws;
  cudaStream_t s = c.s;
  char* scratch = ws + scratch_off;
  const size_t scratch_bytes = c.ws_bytes - 256 - scratch_off;
  int rc;

  // level 0: the caller's waveform -> planes (one pass; writes the whole clip slot)
  if (lv[0].planes) {
    rc = tc_pad_split_ex(c.x, c.x_dtype, B, c.L, c.x_pitch, lv[0].pad, lv[0].mode, lv[0].pitch, lv[0].plane,
                         ws + lv[0].pc, s);
    if (rc) return rc;
  }
  for (int i = 0; i < c.n_octaves; ++i) {
    const Lvl2& l = lv[i];
    const FramedProblem p = octave2_problem(c, l, i);
    int route;
    if (octave_tc_ok(p)) {
      // resident bank + tall A blocks + frame phases: one fetch per sample and tile
      std::pair<cudaEvent_t, cudaEvent_t> pr;
      const bool timed = prof_begin(s, &pr);
      rc = launch_octave_tc(p, c.packed[i], s);
      if (timed) prof_end(s, pr);
      route = NNAB_PYR_OCT_KERNEL;
    } else if (l.presplit) {
      rc = run_framed(p, c.packed[i], nullptr, 0, NNAB_PATH_TCGEN05, s);
      route = NNAB_PYR_OCT_DENSE_PLANES;
    } else {
      rc = run_framed(p, c.packed[i], scratch, scratch_bytes, NNAB_PATH_TCGEN05, s);
      route = NNAB_PYR_OCT_DENSE_FP32;
    }
    if (rc) return rc;
    count_route(route);
    if (i == c.n_octaves - 1) break;
    // ---- FIR stage: level i -> level i + 1
    const Lvl2& d = lv[i + 1];
    DecimParams dec{};
    dec.len_out = d.len;
    if (d.planes) {
      const bool refl = d.mode == NNAB_PAD_REFLECT;
      // what the stage's epilogue never writes: everything outside the samples (+ reflect margins)
      rc = tc_zero_slots(ws + d.pc, B, d.pitch, d.plane, refl ? 0 : d.pad,
                         refl ? d.len + 2 * (int64_t)d.pad : d.pad + d.len, s);
      if (rc) return rc;
      dec.pc = ws + d.pc; dec.pc_plane = d.plane; dec.pc_pitch = d.pitch; dec.pc_off = d.pad;
      dec.pc_reflect = refl ? 1 : 0;
    }
    if (d.y32 != SIZE_MAX) { dec.y32 = (float*)(ws + d.y32); dec.y32_pitch = d.y32_pitch; }
    rc = launch_fir_stage_tc(ws + l.pc, B, l.len, l.pitch, l.plane, l.pad, c.lowpass_packed, c.lowpass,
                             FIR_TAPS, dec, s);
    if (rc) return rc;
    count_route(NNAB_PYR_FIR_BANDED);
  }
  count_route(NNAB_PYR_PLAN_GEN2);
  return NNAB_OK;
}

// Octave i of the gen-1 plan: on the level's reflect-padded planes (one frame phase) or on the fp32 level.
static FramedProblem octave1_problem(const PyramidCall& c, const PyrLevel& l, int i) {
  FramedProblem p = octave_problem(c, i, l.len, l.hop, l.mode);
  if (l.presplit) {
    p.presplit = c.ws + l.pc;
  } else if (i == 0 && c.early_factor <= 1) {  // level 0 is the caller's waveform
    p.x = c.x; p.x_dtype = c.x_dtype; p.x_pitch = c.x_pitch;
  } else {
    p.x = c.ws + l.y32; p.x_pitch = l.y32_pitch;
  }
  return p;
}

// FIR stage of the gen-1 plan: planes `src` (level signal at FIR_OFF, zero margins) -> level `dst`.
static FramedProblem fir1_problem(const PyramidCall& c, const void* src, int64_t src_len, int dec,
                                  const PyrLevel& dst) {
  FramedProblem p{};
  p.x = nullptr; p.B = c.B; p.L = src_len; p.x_pitch = 0;
  p.w_re = nullptr; p.w_im = nullptr; p.F = 64; p.K = tc_fir_k(FIR_TAPS, dec); p.hop = 128 * dec;
  p.pad = FIR_OFF; p.pad_mode = NNAB_PAD_CONSTANT; p.scale = nullptr; p.scale_all = 1.f;
  p.fmt = FMT_DECIM; p.eps = 0.f; p.power = 1.f; p.out = nullptr;
  p.T = (dst.len + 127) / 128;
  p.out_bins = 64; p.bin_offset = 0;
  p.presplit = src;
  p.dec.pc = dst.pc != SIZE_MAX ? c.ws + dst.pc : nullptr;
  p.dec.pc_plane = dst.pc_plane; p.dec.pc_pitch = dst.pc_pitch; p.dec.pc_off = dst.pad;
  p.dec.pc_reflect = dst.mode == NNAB_PAD_REFLECT ? 1 : 0;
  p.dec.pf = dst.pf != SIZE_MAX ? c.ws + dst.pf : nullptr;
  p.dec.pf_plane = dst.pf_plane; p.dec.pf_pitch = dst.pf_pitch;
  p.dec.y32 = dst.y32 != SIZE_MAX ? (float*)(c.ws + dst.y32) : nullptr;
  p.dec.y32_pitch = dst.y32_pitch;
  p.dec.len_out = dst.len;
  return p;
}

// Gen-1 plan of a call: as select_fused2, plus the offset of the early FIR stage's input.
static int select_fused(const PyramidCall& c, PyrLevel* lv, size_t* pf_early, size_t* scratch) {
  if (c.n_octaves > 32 || c.B > 65535) return NNAB_EUNSUPPORTED;
  const size_t need = plan_pyramid(c.B, c.L, c.n_octaves, c.early_factor, c.hop, c.widths, 0, c.pad_mode,
                                   lv, pf_early, scratch);
  if (need + 256 > c.ws_bytes) return NNAB_EUNSUPPORTED;
  for (int i = 0; i < c.n_octaves; ++i) {
    if (lv[i].len <= 0 || lv[i].hop <= 0) return NNAB_EINVAL;
    if (frames_of(lv[i].len, lv[i].width, lv[i].hop, lv[i].pad) != c.T) return NNAB_EINVAL;
  }
  if (c.early_factor > 1 && !tc_supported(fir1_problem(c, c.ws + *pf_early, c.L, c.early_factor, lv[0])))
    return NNAB_EUNSUPPORTED;
  for (int i = 0; i < c.n_octaves; ++i) {
    if (!tc_supported(octave1_problem(c, lv[i], i))) return NNAB_EUNSUPPORTED;
    if (i < c.n_octaves - 1 && !tc_supported(fir1_problem(c, c.ws + lv[i].pf, lv[i].len, 2, lv[i + 1])))
      return NNAB_EUNSUPPORTED;
  }
  return NNAB_OK;
}

static int pyramid_fused(const PyramidCall& c, const PyrLevel* lv, size_t pf_early, size_t scratch_off) {
  const int64_t B = c.B;
  char* const ws = c.ws;
  cudaStream_t s = c.s;
  char* scratch = ws + scratch_off;
  const size_t scratch_bytes = c.ws_bytes - 256 - scratch_off;
  int rc;

  // One FIR stage: planes `src` (level signal, zero margins) -> level `dst`
  auto fir_stage = [&](const void* src, int64_t src_len, int dec, const void* fir_packed,
                       const PyrLevel& dst) -> int {
    // parts of the destination buffers the epilogue never writes
    if (dst.pc != SIZE_MAX) {
      const bool refl = dst.mode == NNAB_PAD_REFLECT;
      rc = tc_zero_slots(ws + dst.pc, B, dst.pc_pitch, dst.pc_plane, refl ? 0 : dst.pad,
                         refl ? dst.len + 2 * dst.pad : dst.pad + dst.len, s);
      if (rc) return rc;
    }
    if (dst.pf != SIZE_MAX) {
      rc = tc_zero_slots(ws + dst.pf, B, dst.pf_pitch, dst.pf_plane, FIR_OFF, FIR_OFF + dst.len, s);
      if (rc) return rc;
    }
    rc = run_framed(fir1_problem(c, src, src_len, dec, dst), fir_packed, nullptr, 0, NNAB_PATH_TCGEN05, s);
    if (rc == NNAB_OK) count_route(NNAB_PYR_FIR_DENSE);
    return rc;
  };

  // ---- level 0 ------------------------------------------------------------------------
  if (c.early_factor > 1) {
    rc = tc_pad_split(c.x, c.x_dtype, B, c.L, c.x_pitch, tc_fir_k(FIR_TAPS, c.early_factor),
                      128 * c.early_factor, FIR_OFF, NNAB_PAD_CONSTANT, ws + pf_early, s);
    if (rc) return rc;
    if ((rc = fir_stage(ws + pf_early, c.L, c.early_factor, c.early_packed, lv[0]))) return rc;
  } else {
    if (lv[0].pc != SIZE_MAX && lv[0].pf != SIZE_MAX) {
      // one pass over x: reflect-padded copy for the octave CQT + zero-margin copy for the FIR
      rc = tc_pad_split2(c.x, c.x_dtype, B, c.L, c.x_pitch, lv[0].width, lv[0].hop, lv[0].pad, lv[0].mode,
                         ws + lv[0].pc, tc_fir_k(FIR_TAPS, 2), 256, FIR_OFF, NNAB_PAD_CONSTANT,
                         ws + lv[0].pf, s);
      if (rc) return rc;
    } else if (lv[0].pc != SIZE_MAX) {
      rc = tc_pad_split(c.x, c.x_dtype, B, c.L, c.x_pitch, lv[0].width, lv[0].hop, lv[0].pad, lv[0].mode,
                        ws + lv[0].pc, s);
      if (rc) return rc;
    } else if (lv[0].pf != SIZE_MAX) {
      rc = tc_pad_split(c.x, c.x_dtype, B, c.L, c.x_pitch, tc_fir_k(FIR_TAPS, 2), 256, FIR_OFF,
                        NNAB_PAD_CONSTANT, ws + lv[0].pf, s);
      if (rc) return rc;
    }
  }

  // ---- octaves --------------------------------------------------------------------------
  for (int i = 0; i < c.n_octaves; ++i) {
    const PyrLevel& l = lv[i];
    const FramedProblem p = octave1_problem(c, l, i);
    if (l.presplit) rc = run_framed(p, c.packed[i], nullptr, 0, NNAB_PATH_TCGEN05, s);
    else rc = run_framed(p, c.packed[i], scratch, scratch_bytes, NNAB_PATH_TCGEN05, s);
    if (rc) return rc;
    count_route(l.presplit ? NNAB_PYR_OCT_DENSE_PLANES : NNAB_PYR_OCT_DENSE_FP32);
    if (i < c.n_octaves - 1)
      if ((rc = fir_stage(ws + l.pf, l.len, 2, c.lowpass_packed, lv[i + 1]))) return rc;
  }
  count_route(NNAB_PYR_PLAN_GEN1);
  return NNAB_OK;
}

int nnab_cqt_pyramid_forward(const float* x, int64_t B, int64_t L, int64_t x_pitch, int n_octaves,
                             const float* const* h_k_real, const float* const* h_k_imag,
                             const void* const* h_packed, const int32_t* h_widths, int n_filters,
                             const float* lowpass, const void* lowpass_packed,
                             const float* early_filter, const void* early_packed,
                             int early_factor, int hop, int pad_mode, int n_bins,
                             const float* scale, float scale_all, int out_format, float sqrt_eps,
                             float* out, int64_t T, void* workspace, size_t ws_bytes, int path,
                             void* stream) {
  return nnab_cqt_pyramid_forward_ex(x, NNAB_DTYPE_F32, B, L, x_pitch, n_octaves, h_k_real, h_k_imag, h_packed,
                                     h_widths, n_filters, lowpass, lowpass_packed, early_filter, early_packed,
                                     early_factor, hop, pad_mode, n_bins, scale, scale_all, out_format,
                                     sqrt_eps, out, T, workspace, ws_bytes, path, stream);
}

int nnab_cqt_pyramid_forward_ex(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch,
                                int n_octaves, const float* const* h_k_real, const float* const* h_k_imag,
                                const void* const* h_packed, const int32_t* h_widths, int n_filters,
                                const float* lowpass, const void* lowpass_packed,
                                const float* early_filter, const void* early_packed,
                                int early_factor, int hop, int pad_mode, int n_bins,
                                const float* scale, float scale_all, int out_format, float sqrt_eps,
                                float* out, int64_t T, void* workspace, size_t ws_bytes, int path,
                                void* stream) {
  if (x == nullptr || !dtype_ok(x_dtype) || out == nullptr || h_k_real == nullptr || h_k_imag == nullptr ||
      h_widths == nullptr || lowpass == nullptr || B < 0 || L <= 0 || x_pitch < L ||
      n_octaves <= 0 || n_filters <= 0 || hop <= 0 || n_bins <= 0 || early_factor < 1)
    return NNAB_EINVAL;
  if (early_factor > 1 && early_filter == nullptr) return NNAB_EINVAL;
  if (out_format != NNAB_FMT_MAGNITUDE && out_format != NNAB_FMT_COMPLEX &&
      out_format != NNAB_FMT_PHASE_UNIT)
    return NNAB_EINVAL;
  if (pad_mode != NNAB_PAD_REFLECT && pad_mode != NNAB_PAD_CONSTANT) return NNAB_EINVAL;
  int rc = check_arch();
  if (rc) return rc;
  int max_width = 0;
  for (int i = 0; i < n_octaves; ++i) max_width = h_widths[i] > max_width ? h_widths[i] : max_width;
  const size_t need =
      nnab_cqt_pyramid_workspace_bytes(B, L, n_octaves, early_factor, max_width, hop, path);
  if (need > 0 && (workspace == nullptr || ws_bytes < need)) return NNAB_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  const PyramidCall c{x, x_dtype, B, L, x_pitch, n_octaves, h_k_real, h_k_imag, h_packed, h_widths, n_filters,
                      lowpass, lowpass_packed, early_packed, early_factor, hop, pad_mode, n_bins, scale,
                      scale_all, out_format, sqrt_eps, out, T,
                      (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255), ws_bytes, s};

  // One plan per call, fixed before anything is enqueued: gen-2 (all-tensor-core, one plane set per
  // level), else gen-1 (all-tensor-core, early downsampling and any bank width), else per-octave --
  // the first whose conditions hold, tc_supported of every stage it runs on the dense tensor-core
  // kernel included.  Once chosen, a plan's every error (NNAB_EUNSUPPORTED too) goes to the caller.
  bool all_packed = (path != NNAB_PATH_SIMT) && h_packed != nullptr && lowpass_packed != nullptr &&
                    (early_factor <= 1 || early_packed != nullptr);
  for (int i = 0; all_packed && i < n_octaves; ++i) all_packed = h_packed[i] != nullptr;
  if (all_packed && early_factor <= 1) {
    Lvl2 lv[32];
    size_t scratch = 0;
    rc = select_fused2(c, lv, &scratch);
    if (rc == NNAB_OK) return pyramid_fused2(c, lv, scratch);
    if (rc != NNAB_EUNSUPPORTED) return rc;
  }
  if (all_packed) {
    PyrLevel lv[32];
    size_t pf_early = 0, scratch = 0;
    rc = select_fused(c, lv, &pf_early, &scratch);
    if (rc == NNAB_OK) return pyramid_fused(c, lv, pf_early, scratch);
    if (rc != NNAB_EUNSUPPORTED) return rc;
  }

  // ---- per-octave path: CUDA-core FIR stages, octaves on either kernel family -----------
  // (its FIR stages read the caller's waveform as fp32)
  if (x_dtype != NNAB_DTYPE_F32) return NNAB_EUNSUPPORTED;
  const size_t level_bytes = pyramid_level_bytes(B, L, early_factor);
  char* tc_ws = (char*)workspace + level_bytes;
  const size_t tc_ws_bytes = ws_bytes - level_bytes;
  char* wsp = (char*)workspace;
  const float* cur = static_cast<const float*>(x);
  int64_t cur_len = L, cur_pitch = x_pitch;
  if (early_factor > 1) {
    const int64_t L0 = decimated_len(L, early_factor);
    const int64_t pitch0 = (int64_t)align_up((size_t)L0, 4);
    float* e = (float*)wsp;
    wsp += align_up((size_t)B * pitch0 * sizeof(float), 256);
    if ((rc = launch_fir_decimate(cur, B, L, x_pitch, early_filter, 256, early_factor, e, L0,
                                  pitch0, s)))
      return rc;
    count_route(NNAB_PYR_FIR_SIMT);
    cur = e; cur_len = L0; cur_pitch = pitch0;
  }
  const int64_t half_pitch = (int64_t)align_up((size_t)(cur_len / 2 + 1), 4);
  float* pingpong[2];
  pingpong[0] = (float*)wsp;
  pingpong[1] = (float*)(wsp + align_up((size_t)B * half_pitch * sizeof(float), 256));

  int cur_hop = hop;
  for (int i = 0; i < n_octaves; ++i) {
    if (i > 0) {
      const int64_t nl = decimated_len(cur_len, 2);
      float* dst = pingpong[i & 1];
      if ((rc = launch_fir_decimate(cur, B, cur_len, cur_pitch, lowpass, 256, 2, dst, nl,
                                    half_pitch, s)))
        return rc;
      count_route(NNAB_PYR_FIR_SIMT);
      cur = dst; cur_len = nl; cur_pitch = half_pitch;
      cur_hop /= 2;
    }
    if (cur_hop <= 0 || cur_len <= 0) return NNAB_EINVAL;
    const int width = h_widths[i];
    const int pad = width / 2;
    // get_cqt_complex: reflect padding that torch would reject falls back to zero padding.
    int mode = pad_mode;
    if (mode == NNAB_PAD_REFLECT && pad >= cur_len) mode = NNAB_PAD_CONSTANT;
    if (frames_of(cur_len, width, cur_hop, pad) != T) return NNAB_EINVAL;
    FramedProblem p = octave_problem(c, i, cur_len, cur_hop, mode);
    p.x = cur; p.x_pitch = cur_pitch;
    const void* pk = (h_packed != nullptr) ? h_packed[i] : nullptr;
    if (pk != nullptr && path != NNAB_PATH_SIMT && tc_supported(p) &&
        tc_ws_bytes >= tc_workspace_bytes(B, cur_len, width, cur_hop, pad)) {
      if ((rc = run_framed(p, pk, tc_ws, tc_ws_bytes, NNAB_PATH_TCGEN05, s))) return rc;
      count_route(NNAB_PYR_OCT_TC_LOOP);
    } else {
      if (path == NNAB_PATH_TCGEN05) return NNAB_EALIGN;
      if ((rc = run_framed(p, nullptr, nullptr, 0, NNAB_PATH_SIMT, s))) return rc;
      count_route(NNAB_PYR_OCT_SIMT);
    }
  }
  count_route(NNAB_PYR_PLAN_PER_OCTAVE);
  return NNAB_OK;
}

// ------------------------------------------------------------ streamed pyramid ----
// (a stream's signals and counters: PyrStream, pyr_counts, pyr_ready_frames and pyr_keep in common.cuh)
static bool pyr_stream_init(int n_octaves, const int32_t* widths, int hop, int early_factor, bool gen2,
                            PyrStream* ps) {
  if (n_octaves <= 0 || n_octaves > 32 || widths == nullptr || hop <= 0 || early_factor < 1) return false;
  if (hop % (1 << (n_octaves - 1)) != 0) return false;  // every octave frames at hop / 2^i
  PyrStream& p = *ps;
  p.n_oct = n_octaves;
  p.e = early_factor > 1 ? 1 : 0;
  p.n_sig = n_octaves + p.e;
  p.gen2 = gen2;
  p.c = gen2 ? 130 : 129;
  for (int s = 0; s + 1 < p.n_sig; ++s) p.d[s] = (p.e && s == 0) ? early_factor : 2;
  for (int i = 0; i < n_octaves; ++i) {
    if (widths[i] < 2) return false;
    p.width[i] = widths[i]; p.hop[i] = hop >> i; p.pad[i] = widths[i] / 2;
  }
  // ring bounds (with the 130 of either plan, so the state size does not depend on the plan): a FIR source reads
  // back from row origin 128 d floor(R'/128) - 128, at most 130 + 127 d + 128 samples; an octave from its first
  // unreturned frame, which the slowest octave holds back by at most (130 + need_i) 2^(i - l) samples of level l
  // (need_i = width_i - pad_i)
  size_t off = 0;
  for (int s = 0; s < p.n_sig; ++s) {
    int64_t span = 0;
    if (s + 1 < p.n_sig) span = 130 + 127 * (int64_t)p.d[s] + 128;
    const int l = s - p.e;
    if (l >= 0) {
      int64_t lag = 0;
      for (int i = 0; i < n_octaves; ++i) {
        const int64_t need = p.width[i] - p.pad[i];
        const int64_t a = i >= l ? (130 + need) << (i - l) : need;
        lag = a > lag ? a : lag;
      }
      const int64_t o = p.pad[l] + 1 + lag;
      span = o > span ? o : span;
    }
    p.ring_len[s] = (span + 64 + 63) / 64 * 64;
    p.ring_off[s] = off;
    off += (size_t)p.ring_len[s];
  }
  p.state_floats = off;
  return true;
}

// Plane geometry of octave l's push clip of `len` samples for the octave kernel (gen-2 single-phase levels):
// (clip pitch, plane stride); the pitch is a multiple of lcm(hop, 64), as the kernel's row blocks need.
static void pyr_oct_geom(const PyrStream& p, int l, int64_t B, int64_t len, int64_t* pitch, int64_t* plane) {
  const int h = p.hop[l];
  const int64_t gran = (int64_t)h / gcd64(h, 64) * 64;
  *pitch = (len + gran - 1) / gran * gran;
  const int64_t kpad = (p.width[l] + 63) / 64 * 64;
  const int64_t rows = B * (*pitch / h) + (kpad + h - 1) / h + 1;
  *plane = (rows * h + 255) / 256 * 256;
}

// The whole-clip call's plan for these shapes: gen-2 without early downsampling when every FIR-source bank is
// 256 wide (plan_pyramid2), else gen-1.
static bool pyr_gen2(int n_octaves, const int32_t* widths, int early_factor) {
  if (early_factor > 1) return false;
  for (int i = 0; i + 1 < n_octaves; ++i)
    if (widths[i] / 2 != 128) return false;
  return true;
}

size_t nnab_cqt_pyramid_chunk_state_bytes(int64_t B, int n_octaves, const int32_t* widths, int hop,
                                          int early_factor) {
  PyrStream p;
  if (B < 0 || widths == nullptr || !pyr_stream_init(n_octaves, widths, hop, early_factor, false, &p)) return 0;
  return (size_t)B * p.state_floats * sizeof(float);
}

// ------------------------------------------------------------ pyramid pools ----
// One push of pyramid streams (DESIGN §3.10 "Pyramid pools"): every lane checked by the one-stream rules (pyr_step)
// and the batch-wide geometry of each launch.  A pool's plan comes from its lane table (pyr_pool_plan), a device
// pool's from its fixed geometry (pyr_device_plan), a lock-step push's from its one set of counters (pyr_chunk_plan).
struct PyrPoolPlan {
  int64_t T_max;
  int64_t len_out[33];  // stage s: the most outputs one lane's FIR rows hold from their first row (0: no lane advances)
  int64_t np[33];       // new-sample row pitch of signal s >= 1 (floats)
  int64_t longest[33];  // the most samples one lane keeps of signal s
  size_t table, nbuf[33], scratch, scratch_bytes, total;
};

// Lane `ln` (row `lane`) of a push: its step by the one-stream rules, its descriptors held to them, and the plan's
// T_max, len_out and longest widened to take it.  *T: the frames the lane returns.
static int pyr_plan_lane(const PyrStream& p, const nnab_stream_lane& ln, int64_t lane, int pad_mode, PyrPoolPlan* o,
                         int64_t* T) {
  if (pad_mode != NNAB_PAD_REFLECT && pad_mode != NNAB_PAD_CONSTANT) return NNAB_EINVAL;
  PyrStep st;
  const int rc = pyr_step(p, ln.received, ln.n_carry, ln.frames, ln.n, (int)ln.end, pad_mode, &st);
  if (rc) return rc;
  *T = st.t_end - ln.frames;
  if (*T > o->T_max) o->T_max = *T;
  for (int s = 0; s < p.n_sig; ++s) {
    const PyrLaneSig d = pyr_lane_signal(p, ln, lane, s, pad_mode);
    if (d.R0 != st.R0[s] || d.R1 != st.R1[s] || d.count != *T) return NNAB_EINVAL;  // one set of rules
    if (d.R1 - d.keep > o->longest[s]) o->longest[s] = d.R1 - d.keep;
    if (d.t0 >= 0 && d.fir_len_out > o->len_out[s]) o->len_out[s] = d.fir_len_out;
  }
  return NNAB_OK;
}

// The workspace of a push of n_lanes lanes, the A first of which return frames, from the plan's T_max, len_out:
// the descriptor table, the new samples of every computed signal (row i: lane i's stage outputs from its first
// row), then one scratch reused by the launches in order.
static void pyr_pool_layout(const PyrStream& p, int64_t n_lanes, int64_t A, PyrPoolPlan* o) {
  size_t off = 0;
  o->table = off;
  off += align_up((size_t)(n_lanes > 0 ? n_lanes : 1) * p.n_sig * sizeof(PyrLaneSig), 256);
  for (int s = 1; s < p.n_sig; ++s) {
    o->np[s] = (int64_t)align_up((size_t)(o->len_out[s - 1] > 0 ? o->len_out[s - 1] : 1), 8);
    o->nbuf[s] = off;
    off += align_up((size_t)(n_lanes > 0 ? n_lanes : 1) * o->np[s] * sizeof(float), 256);
  }
  size_t sc = 0;
  for (int s = 0; s < p.n_sig; ++s) {
    const int l = s - p.e;
    if (l >= 0 && A > 0 && o->T_max > 0) {
      const int64_t len = (o->T_max - 1) * p.hop[l] + p.width[l];
      size_t need = tc_workspace_bytes(A, len, p.width[l], p.hop[l], 0);
      if (p.gen2 && p.hop[l] % 8 == 0) {
        int64_t pitch, plane;
        pyr_oct_geom(p, l, A, len, &pitch, &plane);
        need = (size_t)plane * 4 + 256;
      }
      sc = need > sc ? need : sc;
    }
    if (s + 1 < p.n_sig && o->len_out[s] > 0) {
      const int64_t FT = (o->len_out[s] + 127) / 128;
      const int kf = tc_fir_k(FIR_TAPS, p.d[s]);
      const size_t need = p.gen2 ? (size_t)((n_lanes * (FT + 1) + 2) * 256) * 4 + 256
                                 : tc_workspace_bytes(n_lanes, (FT - 1) * 128 * (int64_t)p.d[s] + kf, kf,
                                                      128 * p.d[s], 0);
      sc = need > sc ? need : sc;
    }
  }
  o->scratch = off;
  o->scratch_bytes = sc;
  o->total = off + sc + 512;
}

static int pyr_pool_plan(const PyrStream& p, const nnab_stream_lane* lanes, int64_t n_lanes, int64_t A,
                         int64_t slots, int64_t n, int pad_mode, PyrPoolPlan* o) {
  if (n_lanes < 0 || n_lanes > slots || A < 0 || A > n_lanes || (n_lanes > 0 && lanes == nullptr)) return NNAB_EINVAL;
  std::vector<uint8_t> seen((size_t)slots, 0);
  *o = PyrPoolPlan{};
  for (int64_t i = 0; i < n_lanes; ++i) {
    const nnab_stream_lane& ln = lanes[i];
    if (ln.slot < 0 || ln.slot >= slots || seen[(size_t)ln.slot]) return NNAB_EINVAL;
    if (i > 0 && i != A && ln.slot <= lanes[i - 1].slot) return NNAB_EINVAL;  // ascending within each group
    seen[(size_t)ln.slot] = 1;
    if (ln.n > n || (ln.end != 0 && ln.end != 1)) return NNAB_EINVAL;
    int64_t T;
    const int rc = pyr_plan_lane(p, ln, i, pad_mode, o, &T);
    if (rc) return rc;
    if ((i < A) != (T > 0)) return NNAB_EINVAL;               // the A lanes with frames come first
    if (T == 0 && ln.n == 0 && !ln.end) return NNAB_EINVAL;   // a lane with nothing to do
  }
  pyr_pool_layout(p, n_lanes, A, o);
  return NNAB_OK;
}

size_t nnab_cqt_pyramid_pool_workspace_bytes(const nnab_stream_lane* lanes, int64_t n_lanes, int64_t A,
                                             int64_t T_max, int n_octaves, const int32_t* widths, int hop,
                                             int early_factor, int pad_mode) {
  PyrStream p;
  PyrPoolPlan pl;
  if (widths == nullptr || n_lanes <= 0 ||
      !pyr_stream_init(n_octaves, widths, hop, early_factor, pyr_gen2(n_octaves, widths, early_factor), &p))
    return 0;
  if (pyr_pool_plan(p, lanes, n_lanes, A, 65535, INT64_MAX, pad_mode, &pl) || pl.T_max != T_max) return 0;
  return pl.total;
}

// The pyramid arguments both pool entry points share, checked on the host.
static int pyr_pool_args_ok(int n_octaves, const float* const* h_k_real, const float* const* h_k_imag,
                            const int32_t* h_widths, int n_filters, const float* lowpass, const float* early_filter,
                            int early_factor, int hop, int pad_mode, int n_bins, int out_format) {
  if (h_k_real == nullptr || h_k_imag == nullptr || h_widths == nullptr || lowpass == nullptr || n_octaves <= 0 ||
      n_octaves > 32 || n_filters <= 0 || hop <= 0 || n_bins <= 0 || early_factor < 1 ||
      (early_factor > 1 && early_filter == nullptr))
    return NNAB_EINVAL;
  if (out_format != NNAB_FMT_MAGNITUDE && out_format != NNAB_FMT_COMPLEX && out_format != NNAB_FMT_PHASE_UNIT)
    return NNAB_EINVAL;
  if (pad_mode != NNAB_PAD_REFLECT && pad_mode != NNAB_PAD_CONSTANT) return NNAB_EINVAL;
  return NNAB_OK;
}

// The whole-clip call's all-tensor-core plans need every packed operand and the tensor-core path.
static bool pyr_packed_ok(int n_octaves, const void* const* h_packed, const void* lowpass_packed,
                          const void* early_packed, int early_factor, int path) {
  bool ok = path != NNAB_PATH_SIMT && h_packed != nullptr && lowpass_packed != nullptr &&
            (early_factor <= 1 || early_packed != nullptr);
  for (int i = 0; ok && i < n_octaves; ++i) ok = h_packed[i] != nullptr;
  return ok;
}

// The body of every pyramid push (pool, device pool and lock-step) on the plan `pl`: every signal's octave (on the A
// rows, T_max frames each), its FIR stage (on the n_lanes rows) and its carry, then the mask.  `table` holds the
// (signal, lane) descriptors, which the plan launch(es) have written before pass 1.  Pass 0 checks every launch
// against the kernels' limits on the host (as the whole-clip plan selection does) and enqueues nothing, so a push
// that cannot run returns before anything is enqueued; pass 1 runs them, and a push that returns frames then counts
// its routes as pyramid_fused2 / pyramid_fused count the whole clip's (nnab_stream_route_count).
static int pyr_pool_run(const PyrStream& p, const PyrPoolPlan& pl, const PyramidCall& c, float* ring,
                        const void* chunk, int chunk_dtype, int64_t slots, int64_t chunk_pitch, int64_t n_lanes,
                        PyrLaneSig* table, char* ws, int pass) {
  const int64_t A = c.B, T_max = c.T;
  const cudaStream_t s = c.s;
  char* scratch = ws + pl.scratch;
  int rc;
  int routes[NNAB_PYR_ROUTES] = {};
  routes[p.gen2 ? NNAB_PYR_PLAN_GEN2 : NNAB_PYR_PLAN_GEN1] = 1;
  for (int sg = 0; sg < p.n_sig; ++sg) {
    ChunkSource cs{};
    cs.ring = ring + (size_t)slots * p.ring_off[sg];
    cs.ring_pitch = cs.ring_len = p.ring_len[sg];
    cs.chunk = sg == 0 ? chunk : (const void*)(ws + pl.nbuf[sg]);
    cs.chunk_pitch = sg == 0 ? chunk_pitch : pl.np[sg];
    cs.pad_mode = NNAB_PAD_CONSTANT;
    cs.rows = table + (size_t)sg * n_lanes;
    const int dt = sg == 0 ? chunk_dtype : NNAB_DTYPE_F32;
    const int l = sg - p.e;
    if (l >= 0 && A > 0 && T_max > 0) {
      // octave l: each row from its lane's first unreturned frame, T_max frames, on the whole-clip plan's kernel
      ChunkSource co = cs;
      co.rows_oct = 1;
      co.pad = p.pad[l];
      co.length = (T_max - 1) * p.hop[l] + p.width[l];
      FramedProblem q = octave_problem(c, l, co.length, p.hop[l], c.pad_mode);
      q.pad = 0; q.x_dtype = dt; q.chunk = &co;
      if (p.gen2 && p.hop[l] % 8 == 0) {
        int64_t pitch, plane;
        pyr_oct_geom(p, l, A, co.length, &pitch, &plane);
        FramedProblem qp = q;
        qp.chunk = nullptr;
        qp.presplit = scratch; qp.presplit_t_slots = pitch / p.hop[l]; qp.presplit_plane_stride = plane;
        const bool oct = octave_tc_ok(qp);
        if (pass == 0) {
          if (!oct && !tc_supported(qp)) return NNAB_EUNSUPPORTED;
        } else {
          if ((rc = tc_chunk_split(co, dt, A, pitch, plane, scratch, s))) return rc;
          if (oct) {
            std::pair<cudaEvent_t, cudaEvent_t> pr;
            const bool timed = prof_begin(s, &pr);
            rc = launch_octave_tc(qp, c.packed[l], s);
            if (timed) prof_end(s, pr);
          } else {
            rc = run_framed(qp, c.packed[l], nullptr, 0, NNAB_PATH_TCGEN05, s);
          }
          if (rc) return rc;
          ++routes[oct ? NNAB_PYR_OCT_KERNEL : NNAB_PYR_OCT_DENSE_PLANES];
        }
      } else if (pass == 0) {
        if (!tc_supported(q)) return NNAB_EUNSUPPORTED;
      } else if ((rc = run_framed(q, c.packed[l], scratch, pl.scratch_bytes, NNAB_PATH_TCGEN05, s))) {
        return rc;
      } else {
        ++routes[NNAB_PYR_OCT_DENSE_FP32];
      }
    }
    if (sg + 1 < p.n_sig && pl.len_out[sg] > 0) {
      // stage sg -> sg + 1 on every lane, each row from its lane's first 128-output row (the whole clip's
      // accumulation order); row i of the new-sample buffer holds lane i's outputs from that row on
      const int d = p.d[sg];
      const int64_t FT = (pl.len_out[sg] + 127) / 128;
      ChunkSource cf = cs;
      cf.rows_oct = 0;
      DecimParams dec{};
      dec.len_out = pl.len_out[sg];
      dec.y32 = (float*)(ws + pl.nbuf[sg + 1]);
      dec.y32_pitch = pl.np[sg + 1];
      const void* fir_packed = (p.e && sg == 0) ? c.early_packed : c.lowpass_packed;
      if (p.gen2) {
        if (pass == 1) {
          const int64_t pitch = 256 * (FT + 1), plane = (n_lanes * (FT + 1) + 2) * 256;
          cf.length = pitch;
          if ((rc = tc_chunk_split(cf, dt, n_lanes, pitch, plane, scratch, s))) return rc;
          if ((rc = launch_fir_stage_tc(scratch, n_lanes, 0, pitch, plane, FIR_OFF, fir_packed, c.lowpass,
                                        FIR_TAPS, dec, s, cf.rows)))
            return rc;
          ++routes[NNAB_PYR_FIR_BANDED];
        }
      } else {
        FramedProblem q{};
        q.B = n_lanes; q.x_dtype = dt; q.F = 64; q.K = tc_fir_k(FIR_TAPS, d); q.hop = 128 * d;
        q.L = (FT - 1) * q.hop + q.K; q.pad = 0; q.pad_mode = NNAB_PAD_CONSTANT; q.scale_all = 1.f;
        q.fmt = FMT_DECIM; q.power = 1.f; q.T = FT; q.out_bins = 64;
        q.dec = dec;
        cf.length = q.L;
        q.chunk = &cf;
        if (pass == 0) {
          if (!tc_supported(q)) return NNAB_EUNSUPPORTED;
        } else if ((rc = run_framed(q, fir_packed, scratch, pl.scratch_bytes, NNAB_PATH_TCGEN05, s))) {
          return rc;
        } else {
          ++routes[NNAB_PYR_FIR_DENSE];
        }
      }
    }
    // after this signal's readers: what later pushes read of it, into each lane's slot row of its ring
    if (pass == 1 && (rc = tc_rows_carry(cs, dt, n_lanes, pl.longest[sg], s))) return rc;
  }
  if (pass == 0) return NNAB_OK;
  // frames t >= a row's count were computed from the zeros past its stream: exact zeros
  if ((rc = tc_rows_mask(table, A, c.out, c.n_bins, T_max, format_cols(c.out_format), s))) return rc;
  if (A > 0 && T_max > 0)
    for (int r = 0; r < NNAB_PYR_ROUTES; ++r)
      if (routes[r]) g_stream_pyr[r].fetch_add(routes[r], std::memory_order_relaxed);
  return NNAB_OK;
}

int nnab_cqt_pyramid_pool_forward(void* state, const nnab_stream_lane* lanes, const nnab_stream_lane* d_lanes,
                                  int64_t n_lanes, int64_t A, const void* chunk, int chunk_dtype, int64_t slots,
                                  int64_t n, int64_t chunk_pitch, int n_octaves, const float* const* h_k_real,
                                  const float* const* h_k_imag, const void* const* h_packed,
                                  const int32_t* h_widths, int n_filters, const float* lowpass,
                                  const void* lowpass_packed, const float* early_filter, const void* early_packed,
                                  int early_factor, int hop, int pad_mode, int n_bins, const float* scale,
                                  float scale_all, int out_format, float sqrt_eps, float* out, int64_t T_max,
                                  void* workspace, size_t ws_bytes, int path, void* stream) {
  if (state == nullptr || !dtype_ok(chunk_dtype) || slots < 1 || slots > 65535 || n < 0 ||
      (n > 0 && chunk == nullptr) || chunk_pitch < n || n_lanes < 0 || n_lanes > slots || A < 0 || A > n_lanes ||
      T_max < 0 || (A > 0 && T_max > 0 && out == nullptr) || (n_lanes > 0 && (lanes == nullptr || d_lanes == nullptr)))
    return NNAB_EINVAL;
  int rc = pyr_pool_args_ok(n_octaves, h_k_real, h_k_imag, h_widths, n_filters, lowpass, early_filter, early_factor,
                            hop, pad_mode, n_bins, out_format);
  if (rc) return rc;
  PyrStream p;
  if (!pyr_stream_init(n_octaves, h_widths, hop, early_factor, pyr_gen2(n_octaves, h_widths, early_factor), &p))
    return NNAB_EUNSUPPORTED;
  PyrPoolPlan pl;
  if ((rc = pyr_pool_plan(p, lanes, n_lanes, A, slots, n, pad_mode, &pl))) return rc;
  if (pl.T_max != T_max) return NNAB_EINVAL;
  if (!pyr_packed_ok(n_octaves, h_packed, lowpass_packed, early_packed, early_factor, path)) return NNAB_EUNSUPPORTED;
  if ((rc = check_arch())) return rc;
  if (n_lanes == 0) return NNAB_OK;
  if (workspace == nullptr || ws_bytes < pl.total) return NNAB_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  PyrLaneSig* table = (PyrLaneSig*)(ws + pl.table);
  // the octaves run on the A lanes with frames (rows 0 .. A - 1), T_max frames each
  const PyramidCall c{nullptr, NNAB_DTYPE_F32, A, 0, 0, n_octaves, h_k_real, h_k_imag, h_packed, h_widths,
                      n_filters, lowpass, lowpass_packed, early_packed, early_factor, hop, pad_mode, n_bins, scale,
                      scale_all, out_format, sqrt_eps, out, T_max, ws, ws_bytes, s};
  float* ring = static_cast<float*>(state);
  if ((rc = pyr_pool_run(p, pl, c, ring, chunk, chunk_dtype, slots, chunk_pitch, n_lanes, table, ws, 0))) return rc;
  if ((rc = tc_pyr_pool_plan(p, d_lanes, nnab_stream_lane{}, n_lanes, pad_mode, table, s))) return rc;
  return pyr_pool_run(p, pl, c, ring, chunk, chunk_dtype, slots, chunk_pitch, n_lanes, table, ws, 1);
}

// One lane's plan in the layout of nnab_debug_pyramid_chunk_plan, from its descriptors.
static void pyr_debug_lane(const PyrStream& p, const nnab_stream_lane& ln, int pad_mode, int64_t* o) {
  const int64_t t_end = ln.frames + pyr_lane_signal(p, ln, 0, 0, pad_mode).count;
  int64_t R1[33];
  pyr_counts(p, ln.received + ln.n, (int)ln.end, R1);
  for (int s = 0; s < p.n_sig; ++s) {
    const PyrLaneSig d = pyr_lane_signal(p, ln, 0, s, pad_mode);
    const PyrLaneSig dn = s + 1 < p.n_sig ? pyr_lane_signal(p, ln, 0, s + 1, pad_mode) : d;
    int64_t* r = o + 8 * s;
    r[0] = d.R0; r[1] = d.R1; r[2] = p.ring_len[s];
    r[3] = d.end ? d.R1 : pyr_keep(p, s, R1, t_end);
    r[4] = d.t0 >= 0 ? d.fir_origin : 0;
    r[5] = d.t0;
    r[6] = d.head ? (dn.R1 < 64 ? dn.R1 : 64) : 0;
    r[7] = d.tail ? (dn.R1 - 64 > dn.R0 ? dn.R1 - 64 : dn.R0) : -1;
  }
  o[8 * p.n_sig] = t_end;
}

// ------------------------------------------------------------ lock-step pyramid streams ----
// A push of StreamingPyramid is a pool push of B lanes that share one set of counters, lane b in slot b (row b of
// the chunk and of every ring): its plan is that one lane's, over B rows.
static int pyr_chunk_plan(const PyrStream& p, int64_t B, const nnab_stream_lane& ln, int pad_mode, PyrPoolPlan* o) {
  if (B < 0 || B > 65535) return NNAB_EINVAL;
  *o = PyrPoolPlan{};
  int64_t T;
  const int rc = pyr_plan_lane(p, ln, 0, pad_mode, o, &T);
  if (rc) return rc;
  pyr_pool_layout(p, B, T > 0 ? B : 0, o);
  return NNAB_OK;
}

size_t nnab_cqt_pyramid_chunk_workspace_bytes(int64_t B, int64_t received, int64_t n_carry, int64_t frames,
                                              int64_t n, int flush, int n_octaves, const int32_t* widths,
                                              int hop, int early_factor, int pad_mode) {
  PyrStream p;
  PyrPoolPlan pl;
  if (widths == nullptr ||
      !pyr_stream_init(n_octaves, widths, hop, early_factor, pyr_gen2(n_octaves, widths, early_factor), &p))
    return 0;
  const nnab_stream_lane ln{0, received, n_carry, frames, n, flush ? 1 : 0};
  if (pyr_chunk_plan(p, B, ln, pad_mode, &pl)) return 0;
  return pl.total;
}

int nnab_cqt_pyramid_chunk_forward(void* state, int64_t received, int64_t n_carry, int64_t frames,
                                   const void* chunk, int chunk_dtype, int64_t B, int64_t n, int64_t chunk_pitch,
                                   int flush, int n_octaves, const float* const* h_k_real,
                                   const float* const* h_k_imag, const void* const* h_packed,
                                   const int32_t* h_widths, int n_filters, const float* lowpass,
                                   const void* lowpass_packed, const float* early_filter, const void* early_packed,
                                   int early_factor, int hop, int pad_mode, int n_bins, const float* scale,
                                   float scale_all, int out_format, float sqrt_eps, float* out, int64_t T,
                                   void* workspace, size_t ws_bytes, int path, void* stream) {
  if (state == nullptr || !dtype_ok(chunk_dtype) || (n > 0 && chunk == nullptr) || chunk_pitch < n ||
      (T > 0 && out == nullptr) || T < 0)
    return NNAB_EINVAL;
  int rc = pyr_pool_args_ok(n_octaves, h_k_real, h_k_imag, h_widths, n_filters, lowpass, early_filter, early_factor,
                            hop, pad_mode, n_bins, out_format);
  if (rc) return rc;
  PyrStream p;
  if (!pyr_stream_init(n_octaves, h_widths, hop, early_factor, pyr_gen2(n_octaves, h_widths, early_factor), &p))
    return NNAB_EUNSUPPORTED;
  const nnab_stream_lane ln{0, received, n_carry, frames, n, flush ? 1 : 0};
  PyrPoolPlan pl;
  if ((rc = pyr_chunk_plan(p, B, ln, pad_mode, &pl))) return rc;
  if (T != pl.T_max) return NNAB_EINVAL;
  if (!pyr_packed_ok(n_octaves, h_packed, lowpass_packed, early_packed, early_factor, path)) return NNAB_EUNSUPPORTED;
  if ((rc = check_arch())) return rc;
  if (workspace == nullptr || ws_bytes < pl.total) return NNAB_EWORKSPACE;
  if (B == 0) return NNAB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  PyrLaneSig* table = (PyrLaneSig*)(ws + pl.table);
  // the octaves run on every row when the push returns frames
  const int64_t A = T > 0 ? B : 0;
  const PyramidCall c{nullptr, NNAB_DTYPE_F32, A, 0, 0, n_octaves, h_k_real, h_k_imag, h_packed, h_widths,
                      n_filters, lowpass, lowpass_packed, early_packed, early_factor, hop, pad_mode, n_bins, scale,
                      scale_all, out_format, sqrt_eps, out, T, ws, ws_bytes, s};
  float* ring = static_cast<float*>(state);
  if ((rc = pyr_pool_run(p, pl, c, ring, chunk, chunk_dtype, B, chunk_pitch, B, table, ws, 0))) return rc;
  if ((rc = tc_pyr_pool_plan(p, nullptr, ln, B, pad_mode, table, s))) return rc;
  return pyr_pool_run(p, pl, c, ring, chunk, chunk_dtype, B, chunk_pitch, B, table, ws, 1);
}

int nnab_debug_pyramid_chunk_plan(int64_t received, int64_t n_carry, int64_t frames, int64_t n, int flush,
                                  int n_octaves, const int32_t* widths, int hop, int early_factor, int pad_mode,
                                  int64_t* out) {
  if (out == nullptr) return NNAB_EINVAL;
  PyrStream p;
  PyrPoolPlan pl;
  if (widths == nullptr ||
      !pyr_stream_init(n_octaves, widths, hop, early_factor, pyr_gen2(n_octaves, widths, early_factor), &p))
    return NNAB_EUNSUPPORTED;
  const nnab_stream_lane ln{0, received, n_carry, frames, n, flush ? 1 : 0};
  const int rc = pyr_chunk_plan(p, 1, ln, pad_mode, &pl);
  if (rc) return rc;
  pyr_debug_lane(p, ln, pad_mode, out);
  return NNAB_OK;
}

// ------------------------------------------------------------ device pyramid pools ----
// The fixed geometry of a device pool's push (DESIGN §3.10 "Device pyramid pools"): over every slot's possible
// push of at most `chunk` samples, an end included, the most frames (T_cap), FIR outputs of each stage from the
// lane's first 128-output row (len_out) and samples one signal's carry stores (longest).  For a given total
// t = received + n every one is nonincreasing in `received` (frames, R0 and R0's 128-row all grow with it, and the
// frame bound, R1 and the ring's first kept sample depend on t alone), so the largest comes from the push that
// reaches t with the most samples: n = chunk from received = t - chunk, or n = t from received = 0.  And every one
// is periodic in t once start-up is past: shifting t by P shifts every count of signal s by P / (d_0 ... d_{s-1})
// and the frames by P / (E hop) (E: the early factor, or 1), so with P = lcm(E hop, 128 d_0 ... d_{n-2}) the
// frames, counts and 128-row alignments of every stage all repeat (ready(raw + f E hop) = ready(raw) + f).
// Start-up is past once no clamp of the rules is active: every level holds at least M = 2 max width + 256 + c
// samples (frames past every pad, rows past 128, the FIR read-back past 0), which raw >= (M + c) d_0 ... d_{n-2}
// ensures.  So the sweep runs pyr_step and pyr_lane_signal themselves, with and without an end, on n = chunk over
// received in [0, start-up + P) and on every n <= chunk from received = 0.  A refused end gets the zero lane and
// contributes nothing; a refused push without an end never happens (pyr_stream_init's ring bounds), and the sweep
// returns NNAB_EINVAL if it did.  The caps are a PyrPoolPlan's T_max, len_out and longest.
static int pyr_caps_sweep(const PyrStream& p, int64_t chunk, int pad_mode, PyrPoolPlan* o) {
  int64_t D = 1;
  for (int s = 0; s + 1 < p.n_sig; ++s) D *= p.d[s];
  int max_w = 0;
  for (int i = 0; i < p.n_oct; ++i) max_w = p.width[i] > max_w ? p.width[i] : max_w;
  const int64_t M = 2 * (int64_t)max_w + 256 + p.c;
  const int64_t E = p.e ? p.d[0] : 1;
  const int64_t a = E * p.hop[0], b = 128 * D;
  const int64_t period = a / gcd64(a, b) * b;
  const int64_t sweep = (M + p.c) * D + period;
  *o = PyrPoolPlan{};
  for (int64_t k = -chunk; k < sweep; ++k) {  // k < 0: received 0, n = chunk + k
    const int64_t rec = k < 0 ? 0 : k;
    nnab_stream_lane ln{};
    int64_t R0[33], T;
    pyr_counts(p, rec, 0, R0);
    ln.received = rec;
    ln.frames = pyr_ready_frames(p, R0, pad_mode);
    ln.n_carry = rec - pyr_keep(p, 0, R0, ln.frames);
    ln.n = k < 0 ? chunk + k : chunk;
    for (int end = 0; end < 2; ++end) {
      ln.end = end;
      if (pyr_plan_lane(p, ln, 0, pad_mode, o, &T) != NNAB_OK && !end) return NNAB_EINVAL;
    }
  }
  return NNAB_OK;
}

// pyr_caps_sweep, computed once per geometry for the life of the process (the push checks its T_max against it).
static int pyr_caps(const PyrStream& p, int64_t chunk, int pad_mode, PyrPoolPlan* o) {
  static std::mutex mu;
  static std::vector<std::pair<std::vector<int64_t>, PyrPoolPlan>> memo;
  std::vector<int64_t> key{chunk, pad_mode, p.n_oct, p.e, p.d[0], p.c, p.hop[0]};
  for (int i = 0; i < p.n_oct; ++i) key.push_back(p.width[i]);
  {
    std::lock_guard<std::mutex> g(mu);
    for (const auto& m : memo)
      if (m.first == key) { *o = m.second; return NNAB_OK; }
  }
  const int rc = pyr_caps_sweep(p, chunk, pad_mode, o);
  if (rc) return rc;
  std::lock_guard<std::mutex> g(mu);
  memo.emplace_back(key, *o);
  return NNAB_OK;
}

// A device pool's plan: its caps, every slot a lane (n_lanes = A = slots), and the workspace layout.
static int pyr_device_plan(int64_t slots, int64_t chunk, int n_octaves, const int32_t* widths, int hop,
                           int early_factor, int pad_mode, PyrStream* p, PyrPoolPlan* o) {
  if (slots < 1 || slots > 65535 || chunk < 1 || widths == nullptr ||
      (pad_mode != NNAB_PAD_REFLECT && pad_mode != NNAB_PAD_CONSTANT))
    return NNAB_EINVAL;
  if (!pyr_stream_init(n_octaves, widths, hop, early_factor, pyr_gen2(n_octaves, widths, early_factor), p))
    return NNAB_EUNSUPPORTED;
  const int rc = pyr_caps(*p, chunk, pad_mode, o);
  if (rc) return rc;
  pyr_pool_layout(*p, slots, slots, o);
  return NNAB_OK;
}

int nnab_cqt_pyramid_pool_device_caps(int64_t chunk, int n_octaves, const int32_t* widths, int hop,
                                      int early_factor, int pad_mode, int64_t* caps) {
  if (caps == nullptr) return NNAB_EINVAL;
  PyrStream p;
  PyrPoolPlan pl;
  const int rc = pyr_device_plan(1, chunk, n_octaves, widths, hop, early_factor, pad_mode, &p, &pl);
  if (rc) return rc;
  caps[0] = pl.T_max;
  for (int s = 0; s < p.n_sig; ++s) {
    caps[1 + s] = s + 1 < p.n_sig ? pl.len_out[s] : 0;
    caps[1 + p.n_sig + s] = pl.longest[s];
  }
  return NNAB_OK;
}

size_t nnab_cqt_pyramid_pool_device_workspace_bytes(int64_t slots, int64_t chunk, int n_octaves,
                                                    const int32_t* widths, int hop, int early_factor, int pad_mode) {
  PyrStream p;
  PyrPoolPlan pl;
  if (pyr_device_plan(slots, chunk, n_octaves, widths, hop, early_factor, pad_mode, &p, &pl)) return 0;
  return pl.total;
}

int nnab_cqt_pyramid_pool_device_forward(void* state, int64_t* counters, const int32_t* lengths, const uint8_t* end,
                                         int32_t* errors, int64_t* error_info, int32_t* counts,
                                         nnab_stream_lane* d_lanes, const void* chunk, int chunk_dtype, int64_t slots,
                                         int64_t n, int64_t chunk_pitch, int n_octaves, const float* const* h_k_real,
                                         const float* const* h_k_imag, const void* const* h_packed,
                                         const int32_t* h_widths, int n_filters, const float* lowpass,
                                         const void* lowpass_packed, const float* early_filter,
                                         const void* early_packed, int early_factor, int hop, int pad_mode,
                                         int n_bins, const float* scale, float scale_all, int out_format,
                                         float sqrt_eps, float* out, int64_t T_max, void* workspace, size_t ws_bytes,
                                         int path, void* stream) {
  if (state == nullptr || counters == nullptr || lengths == nullptr || end == nullptr || errors == nullptr ||
      error_info == nullptr || counts == nullptr || d_lanes == nullptr || chunk == nullptr || out == nullptr ||
      !dtype_ok(chunk_dtype) || slots < 1 || slots > 65535 || n < 1 || chunk_pitch < n)
    return NNAB_EINVAL;
  int rc = pyr_pool_args_ok(n_octaves, h_k_real, h_k_imag, h_widths, n_filters, lowpass, early_filter, early_factor,
                            hop, pad_mode, n_bins, out_format);
  if (rc) return rc;
  PyrStream p;
  PyrPoolPlan pl;
  if ((rc = pyr_device_plan(slots, n, n_octaves, h_widths, hop, early_factor, pad_mode, &p, &pl))) return rc;
  if (T_max != pl.T_max) return NNAB_EINVAL;
  if (!pyr_packed_ok(n_octaves, h_packed, lowpass_packed, early_packed, early_factor, path)) return NNAB_EUNSUPPORTED;
  if ((rc = check_arch())) return rc;
  if (workspace == nullptr || ws_bytes < pl.total) return NNAB_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  PyrLaneSig* table = (PyrLaneSig*)(ws + pl.table);
  // every slot is a lane and an octave row: row s of out is slot s, T_cap frames
  const PyramidCall c{nullptr, NNAB_DTYPE_F32, slots, 0, 0, n_octaves, h_k_real, h_k_imag, h_packed, h_widths,
                      n_filters, lowpass, lowpass_packed, early_packed, early_factor, hop, pad_mode, n_bins, scale,
                      scale_all, out_format, sqrt_eps, out, T_max, ws, ws_bytes, s};
  float* ring = static_cast<float*>(state);
  if ((rc = pyr_pool_run(p, pl, c, ring, chunk, chunk_dtype, slots, chunk_pitch, slots, table, ws, 0))) return rc;
  if ((rc = tc_device_pyramid_plan(p, slots, counters, lengths, end, errors, error_info, counts, d_lanes, n, pad_mode,
                                   s)))
    return rc;
  if ((rc = tc_pyr_pool_plan(p, d_lanes, nnab_stream_lane{}, slots, pad_mode, table, s))) return rc;
  return pyr_pool_run(p, pl, c, ring, chunk, chunk_dtype, slots, chunk_pitch, slots, table, ws, 1);
}

int nnab_debug_device_pyramid_plan(int64_t* counters, const int32_t* lengths, const uint8_t* end, int32_t* errors,
                                   int64_t* error_info, int32_t* counts, nnab_stream_lane* lanes, int64_t slots,
                                   int64_t n, int n_octaves, const int32_t* widths, int hop, int early_factor,
                                   int pad_mode) {
  if (counters == nullptr || lengths == nullptr || end == nullptr || errors == nullptr || error_info == nullptr ||
      counts == nullptr || lanes == nullptr || widths == nullptr || slots < 1 || n < 1 ||
      (pad_mode != NNAB_PAD_REFLECT && pad_mode != NNAB_PAD_CONSTANT))
    return NNAB_EINVAL;
  PyrStream p;
  if (!pyr_stream_init(n_octaves, widths, hop, early_factor, pyr_gen2(n_octaves, widths, early_factor), &p))
    return NNAB_EUNSUPPORTED;
  for (int64_t s = 0; s < slots; ++s)
    device_pyramid_slot(s, slots, counters, lengths, end, errors, error_info, counts, lanes, n, p, pad_mode);
  return NNAB_OK;
}

int nnab_debug_pyramid_pool_plan(const nnab_stream_lane* lanes, int64_t n_lanes, int64_t A, int n_octaves,
                                 const int32_t* widths, int hop, int early_factor, int pad_mode, int64_t* out) {
  if (out == nullptr) return NNAB_EINVAL;
  PyrStream p;
  PyrPoolPlan pl;
  if (widths == nullptr ||
      !pyr_stream_init(n_octaves, widths, hop, early_factor, pyr_gen2(n_octaves, widths, early_factor), &p))
    return NNAB_EUNSUPPORTED;
  const int rc = pyr_pool_plan(p, lanes, n_lanes, A, 65535, INT64_MAX, pad_mode, &pl);
  if (rc) return rc;
  for (int64_t i = 0; i < n_lanes; ++i) pyr_debug_lane(p, lanes[i], pad_mode, out + i * (8 * p.n_sig + 1));
  return NNAB_OK;
}

// ----------------------------------------------------------------- inverse STFT ----
static __global__ void istft_scale_kernel(const float* __restrict__ window, float inv_n, int n,
                                          float* __restrict__ scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) scale[i] = window[i] * inv_n;
}

size_t nnab_packed_istft_bytes(int n_fft, int f_in) { return tc_packed_istft_bytes(n_fft, f_in); }

int nnab_pack_istft_basis(const float* kernel_cos, const float* kernel_sin, int n_fft, int f_in,
                          int onesided, void* packed, void* stream) {
  if (kernel_cos == nullptr || kernel_sin == nullptr || packed == nullptr || n_fft <= 0 ||
      f_in <= 0 || f_in > n_fft)
    return NNAB_EINVAL;
  return tc_pack_istft(kernel_cos, kernel_sin, n_fft, f_in, onesided, packed, (cudaStream_t)stream);
}

static size_t istft_ola_bytes(int64_t B, int64_t T, int n_fft, int hop, int64_t* pitch) {
  const int64_t len = n_fft + (int64_t)hop * (T - 1);
  const int64_t p = (int64_t)align_up((size_t)len, 8);
  if (pitch) *pitch = p;
  return align_up((size_t)B * p * sizeof(float), 256);
}

size_t nnab_istft_workspace_bytes(int64_t B, int f_in, int64_t T, int n_fft, int hop) {
  return align_up(tc_istft_planes_bytes(B, T, f_in), 256) + istft_ola_bytes(B, T, n_fft, hop, nullptr) +
         align_up((size_t)n_fft * sizeof(float), 256) + 256;
}

int nnab_istft_forward(const float* X, int64_t B, int f_in, int64_t T, const void* packed,
                       const float* window, int n_fft, int hop, int center, int64_t length,
                       float* out, int64_t out_len, void* workspace, size_t ws_bytes,
                       void* stream) {
  if (X == nullptr || packed == nullptr || window == nullptr || out == nullptr || B < 0 ||
      f_in <= 0 || T <= 0 || n_fft <= 0 || hop <= 0)
    return NNAB_EINVAL;
  if (!tc_ola_plan(n_fft, tc_istft_k(f_in), B * T, TC_OLA_MAX_SPLITS).supported) return NNAB_EUNSUPPORTED;
  int rc = check_arch();
  if (rc) return rc;
  const size_t need = nnab_istft_workspace_bytes(B, f_in, T, n_fft, hop);
  if (workspace == nullptr || ws_bytes < need) return NNAB_EWORKSPACE;
  const int64_t ola_len = n_fft + (int64_t)hop * (T - 1);
  const int pad = n_fft / 2;
  const int64_t offset = center ? pad : 0;
  int64_t want = length >= 0 ? length : (center ? ola_len - 2 * pad : ola_len);
  if (offset + want > ola_len) want = ola_len - offset;  // slicing past the end just truncates
  if (want < 0) want = 0;
  if (out_len != want) return NNAB_EINVAL;
  if (B == 0 || want == 0) return NNAB_OK;
  cudaStream_t s = (cudaStream_t)stream;

  char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  void* planes = ws;
  int64_t ola_pitch = 0;
  const size_t planes_b = align_up(tc_istft_planes_bytes(B, T, f_in), 256);
  const size_t ola_b = istft_ola_bytes(B, T, n_fft, hop, &ola_pitch);
  float* ola = (float*)(ws + planes_b);
  float* scale = (float*)(ws + planes_b + ola_b);

  if ((rc = tc_istft_prep(X, B, f_in, T, planes, s))) return rc;
  NNAB_CUDA_TRY(cudaMemsetAsync(ola, 0, (size_t)B * ola_pitch * sizeof(float), s));
  istft_scale_kernel<<<(n_fft + 255) / 256, 256, 0, s>>>(window, 1.0f / (float)n_fft, n_fft, scale);
  NNAB_LAUNCH_CHECK();

  const int kpad = tc_istft_k(f_in);
  FramedProblem p{};
  p.x = nullptr; p.B = B; p.L = T * (int64_t)kpad; p.x_pitch = 0;
  p.F = n_fft; p.K = kpad; p.hop = kpad; p.pad = 0; p.pad_mode = NNAB_PAD_CONSTANT;
  p.scale = scale; p.scale_all = 1.f; p.fmt = FMT_OLA; p.eps = 0.f; p.power = 1.f;
  p.out = ola; p.T = T; p.out_bins = n_fft; p.bin_offset = 0;
  p.presplit = planes;
  p.ola_pitch = ola_pitch; p.ola_hop = hop;
  p.k_splits_hint = TC_OLA_MAX_SPLITS;
  if ((rc = run_framed(p, packed, nullptr, 0, NNAB_PATH_TCGEN05, s))) return rc;
  return tc_istft_finalize(ola, ola_pitch, B, window, n_fft, hop, T, offset, out, want, s);
}

// ---- streamed inverse STFT and inverse STFT pools (DESIGN §3.10 "Inverse pools") ---------------------------
// Row i of a push's overlap-add buffer starts `lead` = n_fft positions before lane i's first new frame, so the
// carried sums (at most n_fft / 2 before it) fit and the new frames of every lane start at column `lead`.
static int64_t istft_pool_ola_pitch(int64_t T_max, int n_fft, int hop) {
  const int64_t T = T_max > 0 ? T_max : 1;
  return (int64_t)align_up((size_t)(2 * (int64_t)n_fft + (int64_t)hop * (T - 1)), 8);
}

static int istft_pool_run(float* carry, const nnab_istft_lane* d_lanes, const nnab_istft_lane& shared,
                          int64_t n_lanes, int64_t A, const float* X, int f_in, int64_t t, const void* packed,
                          const float* window, int n_fft, int hop, int center, float* out, int64_t n_max,
                          int64_t T_max, void* workspace, cudaStream_t s);

size_t nnab_istft_pool_workspace_bytes(int64_t n_lanes, int f_in, int64_t T_max, int n_fft, int hop) {
  if (n_lanes <= 0) return 0;
  return nnab_istft_workspace_bytes(n_lanes, f_in, T_max > 0 ? T_max : 1, n_fft, hop) +
         align_up((size_t)n_lanes * align_up((size_t)n_fft, 8) * sizeof(float), 256);
}

size_t nnab_istft_chunk_workspace_bytes(int64_t B, int f_in, int64_t T, int n_fft, int hop) {
  return nnab_istft_pool_workspace_bytes(B, f_in, T, n_fft, hop);
}

// A lock-step push: the pool push of B lanes that share these counters, lane b in slot b and X row b.
int nnab_istft_chunk_forward(void* state, int64_t frames, int64_t emitted, const float* X, int64_t B, int f_in,
                             int64_t T, const void* packed, const float* window, int n_fft, int hop, int center,
                             int flush, int64_t length, float* out, int64_t out_len, void* workspace,
                             size_t ws_bytes, void* stream) {
  if (state == nullptr || (T > 0 && X == nullptr) || packed == nullptr || window == nullptr || B < 0 ||
      B > 65535 || f_in <= 0)
    return NNAB_EINVAL;
  IstftChunkPlan pl;
  int rc = istft_chunk_plan(frames, emitted, T, n_fft, hop, center, flush, length, &pl);
  if (rc) return rc;
  const int64_t n_out = pl.emit_end - pl.emit_begin;
  if (out_len != n_out || (n_out > 0 && out == nullptr)) return NNAB_EINVAL;
  if ((rc = check_arch())) return rc;
  const size_t need = nnab_istft_chunk_workspace_bytes(B, f_in, T, n_fft, hop);
  if (workspace == nullptr || ws_bytes < need) return NNAB_EWORKSPACE;
  if (B == 0 || (T == 0 && n_out == 0)) return NNAB_OK;  // nothing new: the carry stays as it is
  const nnab_istft_lane ln{0, 0, frames, emitted, T, flush ? 1 : 0, length};
  return istft_pool_run(static_cast<float*>(state), nullptr, ln, B, n_out > 0 ? B : 0, X, f_in, T, packed, window,
                        n_fft, hop, center, out, n_out, T, workspace, (cudaStream_t)stream);
}

int nnab_istft_pool_forward(void* state, const nnab_istft_lane* lanes, const nnab_istft_lane* d_lanes,
                            int64_t n_lanes, int64_t A, int64_t slots, const float* X, int64_t R, int f_in, int64_t t,
                            const void* packed, const float* window, int n_fft, int hop, int center, float* out,
                            int64_t n_max, int64_t T_max, void* workspace, size_t ws_bytes, void* stream) {
  if (state == nullptr || packed == nullptr || window == nullptr || slots < 1 || slots > 65535 || n_lanes < 0 ||
      n_lanes > slots || A < 0 || A > n_lanes || R < 0 || t < 0 || f_in <= 0 || n_max < 0 || T_max < 0 ||
      (n_lanes > 0 && (lanes == nullptr || d_lanes == nullptr)))
    return NNAB_EINVAL;
  // every lane by istft_chunk_plan, then the table's order, rows and totals, before anything runs
  std::vector<uint8_t> seen((size_t)slots, 0), used((size_t)R, 0);
  int64_t n_most = 0, t_most = 0;
  for (int64_t i = 0; i < n_lanes; ++i) {
    const nnab_istft_lane& ln = lanes[i];
    if (ln.slot < 0 || ln.slot >= slots || seen[(size_t)ln.slot]) return NNAB_EINVAL;
    if (i > 0 && i != A && ln.slot <= lanes[i - 1].slot) return NNAB_EINVAL;  // ascending within each group
    seen[(size_t)ln.slot] = 1;
    if (ln.T < 0 || ln.T > t || (ln.end != 0 && ln.end != 1)) return NNAB_EINVAL;
    if ((ln.row < 0) != (ln.T == 0)) return NNAB_EINVAL;  // a row exactly for the lanes with frames
    if (ln.row >= 0) {
      if (ln.row >= R || used[(size_t)ln.row]) return NNAB_EINVAL;
      used[(size_t)ln.row] = 1;
    }
    if (ln.T == 0 && !ln.end) return NNAB_EINVAL;  // a lane with nothing to do
    IstftChunkPlan pl;
    const int rc = istft_chunk_plan(ln.frames, ln.emitted, ln.T, n_fft, hop, center, (int)ln.end,
                                    ln.end ? ln.length : -1, &pl);
    if (rc) return rc;
    const int64_t n_out = pl.emit_end - pl.emit_begin;
    if ((i < A) != (n_out > 0)) return NNAB_EINVAL;  // the A lanes with samples come first
    if (n_out > n_most) n_most = n_out;
    if (ln.T > t_most) t_most = ln.T;
  }
  if (n_most != n_max || t_most != T_max) return NNAB_EINVAL;
  if ((t_most > 0 && X == nullptr) || (A > 0 && out == nullptr)) return NNAB_EINVAL;
  int rc = check_arch();
  if (rc) return rc;
  const size_t need = nnab_istft_pool_workspace_bytes(n_lanes, f_in, T_max, n_fft, hop);
  if (n_lanes > 0 && (workspace == nullptr || ws_bytes < need)) return NNAB_EWORKSPACE;
  if (n_lanes == 0) return NNAB_OK;
  return istft_pool_run(static_cast<float*>(state), d_lanes, nnab_istft_lane{}, n_lanes, A, X, f_in, t, packed,
                        window, n_fft, hop, center, out, n_max, T_max, workspace, (cudaStream_t)stream);
}

// The launches of an inverse push on checked lanes (seed, pre-pass and GEMM, finalize): the DEVICE lane table
// d_lanes, or without one `shared` in slot i with X row i.
static int istft_pool_run(float* carry, const nnab_istft_lane* d_lanes, const nnab_istft_lane& shared,
                          int64_t n_lanes, int64_t A, const float* X, int f_in, int64_t t, const void* packed,
                          const float* window, int n_fft, int hop, int center, float* out, int64_t n_max,
                          int64_t T_max, void* workspace, cudaStream_t s) {
  int rc;
  // nnab_istft_forward's layout for n_lanes x max(T_max, 1) frames, each row `lead` positions longer
  const int64_t lead = n_fft;
  const int64_t ola_pitch = istft_pool_ola_pitch(T_max, n_fft, hop);
  char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  void* planes = ws;
  const size_t planes_b = align_up(tc_istft_planes_bytes(n_lanes, T_max > 0 ? T_max : 1, f_in), 256);
  const size_t ola_b = align_up((size_t)n_lanes * ola_pitch * sizeof(float), 256);
  float* ola = (float*)(ws + planes_b);
  float* scale = (float*)(ws + planes_b + ola_b);

  // 1. every row: its carried sums where they lie, zeros elsewhere
  if ((rc = tc_istft_pool_seed(d_lanes, shared, n_lanes, carry, n_fft, hop, center, lead, ola, ola_pitch, s)))
    return rc;
  // 2. the new frames of every lane, overlap-added from column `lead` (one FMT_OLA GEMM over n_lanes x T_max)
  if (T_max > 0) {
    if ((rc = tc_istft_pool_prep(X, d_lanes, n_lanes, f_in, T_max, t, planes, s))) return rc;
    istft_scale_kernel<<<(n_fft + 255) / 256, 256, 0, s>>>(window, 1.0f / (float)n_fft, n_fft, scale);
    NNAB_LAUNCH_CHECK();
    const int kpad = tc_istft_k(f_in);
    FramedProblem p{};
    p.x = nullptr; p.B = n_lanes; p.L = T_max * (int64_t)kpad; p.x_pitch = 0;
    p.F = n_fft; p.K = kpad; p.hop = kpad; p.pad = 0; p.pad_mode = NNAB_PAD_CONSTANT;
    p.scale = scale; p.scale_all = 1.f; p.fmt = FMT_OLA; p.eps = 0.f; p.power = 1.f;
    p.out = ola + lead; p.T = T_max; p.out_bins = n_fft; p.bin_offset = 0;
    p.presplit = planes;
    p.ola_pitch = ola_pitch; p.ola_hop = hop;
    p.k_splits_hint = TC_OLA_MAX_SPLITS;  // K chunks of nnab_istft_forward: <= 4096 products per fp32 accumulator
    if ((rc = run_framed(p, packed, nullptr, 0, NNAB_PATH_TCGEN05, s))) return rc;
  }
  // 3. every lane's final samples / window sum-square (rows i < A of out, zeros up to n_max), its tail carried
  return tc_istft_pool_finalize(d_lanes, shared, n_lanes, A, ola, ola_pitch, lead, window, n_fft, hop, center, out,
                                n_max, carry, s);
}

// ---- device pools (DESIGN §3.10 "Device pools") -----------------------------------------------------------
// n_cap: a push of `frames` frames returns the most samples on a flush with the longest length, after enough
// frames that neither the centre crop nor the earliest possible end hold any back: the whole overlap-add span of
// the new frames past the first returned position, hop * frames + max(n_fft - hop, offset).  Pushes before the
// end return at most hop * frames.
int64_t nnab_istft_pool_sample_cap(int64_t frames, int n_fft, int hop, int center) {
  if (frames < 1 || n_fft <= 0 || hop <= 0 || hop > n_fft) return 0;
  const int64_t offset = center ? n_fft / 2 : 0;
  return (int64_t)hop * frames + (n_fft - hop > offset ? n_fft - hop : offset);
}

int nnab_istft_pool_device_forward(void* state, int64_t* counters, const int32_t* frame_counts, const uint8_t* end,
                                   const int64_t* length, int32_t* errors, int64_t* error_info, int32_t* counts,
                                   nnab_istft_lane* d_lanes, int64_t slots, const float* X, int f_in, int64_t t,
                                   const void* packed, const float* window, int n_fft, int hop, int center,
                                   float* out, int64_t n_max, void* workspace, size_t ws_bytes, void* stream) {
  if (state == nullptr || counters == nullptr || frame_counts == nullptr || end == nullptr || length == nullptr ||
      errors == nullptr || error_info == nullptr || counts == nullptr || d_lanes == nullptr || X == nullptr ||
      packed == nullptr || window == nullptr || out == nullptr || slots < 1 || slots > 65535 || f_in <= 0 || t < 1 ||
      n_max != nnab_istft_pool_sample_cap(t, n_fft, hop, center))
    return NNAB_EINVAL;
  int rc = check_arch();
  if (rc) return rc;
  if (workspace == nullptr || ws_bytes < nnab_istft_pool_workspace_bytes(slots, f_in, t, n_fft, hop))
    return NNAB_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  if ((rc = tc_device_istft_plan(slots, counters, frame_counts, end, length, errors, error_info, counts, d_lanes, t,
                                 n_fft, hop, center, s)))
    return rc;
  return istft_pool_run(static_cast<float*>(state), d_lanes, nnab_istft_lane{}, slots, slots, X, f_in, t, packed,
                        window, n_fft, hop, center, out, n_max, t, workspace, s);
}

int nnab_pool_device_reset(int64_t* counters, int32_t* errors, int64_t* error_info, const uint8_t* mask,
                           int64_t slots, void* stream) {
  if (counters == nullptr || errors == nullptr || error_info == nullptr || slots < 1 || slots > 65535)
    return NNAB_EINVAL;
  const int rc = check_arch();
  if (rc) return rc;
  return tc_device_pool_reset(slots, counters, errors, error_info, mask, (cudaStream_t)stream);
}

int nnab_debug_device_pool_plan(int64_t* counters, const int32_t* lengths, const uint8_t* end, int32_t* errors,
                                int64_t* error_info, int32_t* counts, nnab_stream_lane* lanes, int64_t slots,
                                int64_t n, int K, int hop, int pad, int pad_mode) {
  if (counters == nullptr || lengths == nullptr || end == nullptr || errors == nullptr || error_info == nullptr ||
      counts == nullptr || lanes == nullptr || slots < 1 || n < 1 || K < 2 || hop <= 0 || pad < 0 || 2 * pad > K ||
      (pad_mode != NNAB_PAD_REFLECT && pad_mode != NNAB_PAD_CONSTANT))
    return NNAB_EINVAL;
  for (int64_t s = 0; s < slots; ++s)
    device_pool_slot(s, slots, counters, lengths, end, errors, error_info, counts, lanes, n, K, hop, pad, pad_mode);
  return NNAB_OK;
}

int nnab_debug_device_istft_plan(int64_t* counters, const int32_t* frame_counts, const uint8_t* end,
                                 const int64_t* length, int32_t* errors, int64_t* error_info, int32_t* counts,
                                 nnab_istft_lane* lanes, int64_t slots, int64_t t, int n_fft, int hop, int center) {
  if (counters == nullptr || frame_counts == nullptr || end == nullptr || length == nullptr || errors == nullptr ||
      error_info == nullptr || counts == nullptr || lanes == nullptr || slots < 1 || t < 1 || n_fft <= 0 ||
      hop <= 0 || hop > n_fft)
    return NNAB_EINVAL;
  for (int64_t s = 0; s < slots; ++s)
    device_istft_slot(s, slots, counters, frame_counts, end, length, errors, error_info, counts, lanes, t, n_fft,
                      hop, center);
  return NNAB_OK;
}

// ------------------------------------------------------------- input gradient ----
size_t nnab_packed_adjoint_bytes(int K, int F) { return tc_packed_istft_bytes(K, F); }

int nnab_pack_adjoint_basis(const float* w_re, const float* w_im, int F, int K, void* packed,
                            void* stream) {
  if (w_re == nullptr || w_im == nullptr || packed == nullptr || F <= 0 || K <= 0) return NNAB_EINVAL;
  return tc_pack_istft(w_re, w_im, K, F, 0, packed, (cudaStream_t)stream, /*transposed=*/1);
}

size_t nnab_framed_backward_input_workspace_bytes(int64_t B, int64_t L, int K, int F, int hop,
                                                  int center) {
  const int pad = center ? K / 2 : 0;
  const int64_t T = frames_of(L, K, hop, pad);
  const int64_t pitch = (int64_t)align_up((size_t)(L + 2 * (int64_t)pad + K), 8);
  return align_up(tc_istft_planes_bytes(B, T, F), 256) +
         align_up((size_t)B * pitch * sizeof(float), 256) + 256;
}

int nnab_framed_backward_input(const float* g, int64_t B, int F, int64_t T, const void* packed_adj,
                               int K, int hop, int center, int pad_mode, float* dx, int64_t L,
                               void* workspace, size_t ws_bytes, void* stream) {
  if (g == nullptr || packed_adj == nullptr || dx == nullptr || B < 0 || F <= 0 || K <= 0 ||
      hop <= 0 || L <= 0)
    return NNAB_EINVAL;
  const int pad = center ? K / 2 : 0;
  if (T != frames_of(L, K, hop, pad) || T <= 0) return NNAB_EINVAL;
  if (!tc_ola_plan(K, tc_istft_k(F), B * T, TC_OLA_MAX_SPLITS).supported) return NNAB_EUNSUPPORTED;
  int rc = check_arch();
  if (rc) return rc;
  const size_t need = nnab_framed_backward_input_workspace_bytes(B, L, K, F, hop, center);
  if (workspace == nullptr || ws_bytes < need) return NNAB_EWORKSPACE;
  if (B == 0) return NNAB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  void* planes = ws;
  const size_t planes_b = align_up(tc_istft_planes_bytes(B, T, F), 256);
  const int64_t gp_len = L + 2 * (int64_t)pad;
  const int64_t pitch = (int64_t)align_up((size_t)(gp_len + K), 8);
  float* gp = (float*)(ws + planes_b);

  if ((rc = tc_istft_prep(g, B, F, T, planes, s))) return rc;
  NNAB_CUDA_TRY(cudaMemsetAsync(gp, 0, (size_t)B * pitch * sizeof(float), s));
  const int kpad = tc_istft_k(F);
  FramedProblem p{};
  p.x = nullptr; p.B = B; p.L = T * (int64_t)kpad; p.x_pitch = 0;
  p.F = K; p.K = kpad; p.hop = kpad; p.pad = 0; p.pad_mode = NNAB_PAD_CONSTANT;
  p.scale = nullptr; p.scale_all = 1.f; p.fmt = FMT_OLA; p.eps = 0.f; p.power = 1.f;
  p.out = gp; p.T = T; p.out_bins = K; p.bin_offset = 0;
  p.presplit = planes;
  p.ola_pitch = pitch; p.ola_hop = hop;
  p.k_splits_hint = TC_OLA_MAX_SPLITS;
  if ((rc = run_framed(p, packed_adj, nullptr, 0, NNAB_PATH_TCGEN05, s))) return rc;
  return tc_unpad_adjoint(gp, pitch, gp_len, B, pad, pad_mode, L, dx, s);
}

size_t nnab_framed_backward_weight_workspace_bytes(int64_t B, int64_t L, int K, int F, int hop,
                                                   int center) {
  const int pad = center ? K / 2 : 0;
  const int64_t T = frames_of(L, K, hop, pad);
  return align_up(tc_dw_grad_planes_bytes(B, T, F), 256) + align_up(tc_dw_frames_bytes(B, T, K), 256) +
         512;
}

int nnab_framed_backward_weight(const float* g, const float* x, int64_t B, int64_t L,
                                int64_t x_pitch, int F, int64_t T, int K, int hop, int center,
                                int pad_mode, float* dw, void* workspace, size_t ws_bytes,
                                void* stream) {
  if (g == nullptr || x == nullptr || dw == nullptr || B <= 0 || L <= 0 || x_pitch < L || F <= 0 ||
      K <= 0 || hop <= 0)
    return NNAB_EINVAL;
  const int pad = center ? K / 2 : 0;
  if (T != frames_of(L, K, hop, pad) || T <= 0) return NNAB_EINVAL;
  const int64_t gpad = tc_dw_gpad(B, T);
  if (gpad >= (1ll << 31)) return NNAB_EUNSUPPORTED;
  if (!tc_ola_plan(K, (int)gpad, 2 * (int64_t)F, TC_OLA_MAX_SPLITS).supported) return NNAB_EUNSUPPORTED;
  int rc = check_arch();
  if (rc) return rc;
  const size_t need = nnab_framed_backward_weight_workspace_bytes(B, L, K, F, hop, center);
  if (workspace == nullptr || ws_bytes < need) return NNAB_EWORKSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  void* gplanes = ws;
  void* frames = ws + align_up(tc_dw_grad_planes_bytes(B, T, F), 256);

  if ((rc = tc_dw_prep_grad(g, B, F, T, gplanes, s))) return rc;
  if ((rc = tc_dw_prep_frames(x, B, L, x_pitch, K, hop, pad, pad_mode, T, frames, s))) return rc;
  NNAB_CUDA_TRY(cudaMemsetAsync(dw, 0, (size_t)2 * F * K * sizeof(float), s));

  FramedProblem p{};
  p.x = nullptr; p.B = 1; p.L = (int64_t)2 * F * gpad; p.x_pitch = 0;
  p.F = K; p.K = (int)gpad; p.hop = (int)gpad; p.pad = 0; p.pad_mode = NNAB_PAD_CONSTANT;
  p.scale = nullptr; p.scale_all = 1.f; p.fmt = FMT_OLA; p.eps = 0.f; p.power = 1.f;
  p.out = dw; p.T = 2 * F; p.out_bins = K; p.bin_offset = 0;
  p.presplit = gplanes;
  p.ola_pitch = 0; p.ola_hop = K;        // row m of dW starts at m * K
  p.k_splits_hint = TC_OLA_MAX_SPLITS;  // <= 64 k-blocks per accumulator chunk
  return run_framed(p, frames, nullptr, 0, NNAB_PATH_TCGEN05, s);
}

// ------------------------------------------------------------ chunked streams ----
size_t nnab_chunk_state_bytes(int64_t B, int K) {
  return (B <= 0 || K <= 0) ? 0 : (size_t)B * K * sizeof(float);
}

size_t nnab_stft_chunk_workspace_bytes(int64_t B, int64_t received, int64_t frames, int64_t n, int flush,
                                       int n_fft, int F, int hop, int center, int pad_mode, int path) {
  const int64_t T = chunk_frames(received, frames, n, flush, n_fft, hop, center ? n_fft / 2 : 0, pad_mode);
  return nnab_stft_pool_workspace_bytes(T > 0 ? B : 0, T, n_fft, F, hop, path);
}

int nnab_stft_chunk_forward(void* state, int64_t received, int64_t n_carry, int64_t frames, const void* chunk,
                            int chunk_dtype, int64_t B, int64_t n, int64_t chunk_pitch, int flush,
                            const float* wcos, const float* wsin, const void* packed, int n_fft, int F, int hop,
                            int center, int pad_mode, int out_format, float sqrt_eps, float* out, int64_t T,
                            void* workspace, size_t ws_bytes, int path, void* stream) {
  PoolPlan pp;
  int rc = lock_step_plan(state, received, n_carry, frames, chunk, chunk_dtype, B, n, chunk_pitch, flush, n_fft, hop,
                          center ? n_fft / 2 : 0, pad_mode, &pp);
  if (rc) return rc;
  if (T != pp.T_max || F <= 0 || (T > 0 && out == nullptr) || stft_args_ok(wcos, wsin, out_format))
    return NNAB_EINVAL;
  int routes[2] = {-1, -1};  // stays -1 when nothing was enqueued
  rc = pool_forward(pp, chunk_dtype, B, out, F, format_cols(out_format), [&](const Wave& w, cudaStream_t s) {
    return stft_run(w, wcos, wsin, packed, n_fft, F, hop, out_format, sqrt_eps, out, T, workspace,
                    ws_bytes, path, s, &routes[0]);
  }, stream);
  if (rc == NNAB_OK) count_stft_routes(routes, g_stream_stft);
  return rc;
}

size_t nnab_filterbank_chunk_workspace_bytes(int64_t B, int64_t received, int64_t frames, int64_t n, int flush,
                                             int n_fft, int F, int hop, int center, int pad_mode, int n_fb,
                                             int path, int has_table) {
  const int64_t T = chunk_frames(received, frames, n, flush, n_fft, hop, center ? n_fft / 2 : 0, pad_mode);
  return nnab_filterbank_pool_workspace_bytes(T > 0 ? B : 0, T, n_fft, F, hop, n_fb, path, has_table);
}

int nnab_stft_filterbank_chunk_forward(void* state, int64_t received, int64_t n_carry, int64_t frames,
                                       const void* chunk, int chunk_dtype, int64_t B, int64_t n,
                                       int64_t chunk_pitch, int flush, const float* wcos, const float* wsin,
                                       const void* packed, int n_fft, int F, int hop, int center, int pad_mode,
                                       float sqrt_eps, float power, const float* fb, int n_fb,
                                       const void* fb_table, float* out, int64_t T, void* workspace,
                                       size_t ws_bytes, int path, void* stream) {
  PoolPlan pp;
  int rc = lock_step_plan(state, received, n_carry, frames, chunk, chunk_dtype, B, n, chunk_pitch, flush, n_fft, hop,
                          center ? n_fft / 2 : 0, pad_mode, &pp);
  if (rc) return rc;
  if (T != pp.T_max || F <= 0 || (T > 0 && out == nullptr) || filterbank_args_ok(wcos, wsin, fb, n_fb))
    return NNAB_EINVAL;
  int routes[2] = {-1, -1};
  rc = pool_forward(pp, chunk_dtype, B, out, n_fb, 1, [&](const Wave& w, cudaStream_t s) {
    return filterbank_run(w, wcos, wsin, packed, n_fft, F, hop, sqrt_eps, power, fb, n_fb, fb_table, out, T,
                          workspace, ws_bytes, path, s, &routes);
  }, stream);
  if (rc == NNAB_OK) count_stft_routes(routes, g_stream_stft);
  return rc;
}

size_t nnab_mfcc_chunk_workspace_bytes(int64_t B, int64_t received, int64_t frames, int64_t n, int flush,
                                       int n_fft, int F, int hop, int center, int pad_mode, int n_mels, int path,
                                       int has_table) {
  const int64_t T = chunk_frames(received, frames, n, flush, n_fft, hop, center ? n_fft / 2 : 0, pad_mode);
  return nnab_mfcc_pool_workspace_bytes(T > 0 ? B : 0, T, n_fft, F, hop, n_mels, path, has_table);
}

int nnab_mfcc_chunk_forward(void* state, int64_t received, int64_t n_carry, int64_t frames, const void* chunk,
                            int chunk_dtype, int64_t B, int64_t n, int64_t chunk_pitch, int flush,
                            const float* wcos, const float* wsin, const void* packed, int n_fft, int F, int hop,
                            int center, int pad_mode, float sqrt_eps, float power, const float* mel_basis,
                            int n_mels, const void* fb_table, float amin, float ref, float top_db,
                            const float* dct, int n_mfcc, float* out, int64_t T, void* workspace,
                            size_t ws_bytes, int path, void* stream) {
  PoolPlan pp;
  int rc = lock_step_plan(state, received, n_carry, frames, chunk, chunk_dtype, B, n, chunk_pitch, flush, n_fft, hop,
                          center ? n_fft / 2 : 0, pad_mode, &pp);
  if (rc) return rc;
  // the top_db floor is a maximum over the whole clip: a stream cannot apply it frame by frame
  if (T != pp.T_max || F <= 0 || (T > 0 && out == nullptr) || top_db >= 0.f ||
      mfcc_args_ok(wcos, wsin, mel_basis, n_mels, dct, n_mfcc, amin))
    return NNAB_EINVAL;
  int routes[2] = {-1, -1};
  rc = pool_forward(pp, chunk_dtype, B, out, n_mfcc, 1, [&](const Wave& w, cudaStream_t s) {
    return mfcc_run(w, wcos, wsin, packed, n_fft, F, hop, sqrt_eps, power, mel_basis, n_mels, fb_table, amin,
                    ref, top_db, dct, n_mfcc, out, T, workspace, ws_bytes, path, s, &routes);
  }, stream);
  if (rc == NNAB_OK) count_stft_routes(routes, g_stream_stft);
  return rc;
}

size_t nnab_cqt1992v2_chunk_workspace_bytes(int64_t B, int64_t received, int64_t frames, int64_t n, int flush,
                                            int width, int n_bins, int hop, int center, int pad_mode, int path) {
  const int64_t T = chunk_frames(received, frames, n, flush, width, hop, center ? width / 2 : 0, pad_mode);
  return nnab_cqt1992v2_pool_workspace_bytes(T > 0 ? B : 0, T, width, n_bins, hop, path);
}

int nnab_cqt1992v2_chunk_forward(void* state, int64_t received, int64_t n_carry, int64_t frames,
                                 const void* chunk, int chunk_dtype, int64_t B, int64_t n, int64_t chunk_pitch,
                                 int flush, const float* k_real, const float* k_imag, const void* packed,
                                 const int32_t* h_k_begin, const int32_t* h_k_end, int n_bins, int width,
                                 int hop, int center, int pad_mode, const float* scale, float scale_all,
                                 int out_format, float sqrt_eps, float* out, int64_t T, void* workspace,
                                 size_t ws_bytes, int path, void* stream) {
  PoolPlan pp;
  int rc = lock_step_plan(state, received, n_carry, frames, chunk, chunk_dtype, B, n, chunk_pitch, flush, width, hop,
                          center ? width / 2 : 0, pad_mode, &pp);
  if (rc) return rc;
  if (T != pp.T_max || n_bins <= 0 || (T > 0 && out == nullptr) || cqt1992v2_args_ok(k_real, k_imag, out_format))
    return NNAB_EINVAL;
  int route = -1;
  rc = pool_forward(pp, chunk_dtype, B, out, n_bins, format_cols(out_format), [&](const Wave& w, cudaStream_t s) {
    return cqt1992v2_run(w, k_real, k_imag, packed, h_k_begin, h_k_end, n_bins, width, hop, scale, scale_all,
                         out_format, sqrt_eps, out, T, workspace, ws_bytes, path, s, &route);
  }, stream);
  if (rc == NNAB_OK) count_cq1992_route(route, g_stream_cq1992);
  return rc;
}

// ------------------------------------------------------------ stream pools ----
size_t nnab_stft_pool_workspace_bytes(int64_t A, int64_t T_max, int n_fft, int F, int hop, int path) {
  const int64_t Lv = pool_clip_length(A, T_max, n_fft, hop);
  return Lv > 0 ? nnab_stft_workspace_bytes(A, Lv, n_fft, F, hop, 0, path) : 0;
}

int nnab_stft_pool_forward(void* state, const nnab_stream_lane* lanes, const nnab_stream_lane* d_lanes,
                           int64_t n_lanes, int64_t A, const void* chunk, int chunk_dtype, int64_t slots, int64_t n,
                           int64_t chunk_pitch, const float* wcos, const float* wsin, const void* packed, int n_fft,
                           int F, int hop, int center, int pad_mode, int out_format, float sqrt_eps, float* out,
                           int64_t T_max, void* workspace, size_t ws_bytes, int path, void* stream) {
  PoolPlan pp;
  int rc = pool_plan(state, lanes, d_lanes, n_lanes, A, chunk, chunk_dtype, slots, n, chunk_pitch, n_fft, hop,
                     center ? n_fft / 2 : 0, pad_mode, T_max, &pp);
  if (rc) return rc;
  if (F <= 0 || (A > 0 && out == nullptr) || stft_args_ok(wcos, wsin, out_format)) return NNAB_EINVAL;
  int routes[2] = {-1, -1};  // stays -1 when nothing was enqueued
  rc = pool_forward(pp, chunk_dtype, n_lanes, out, F, format_cols(out_format),
                      [&](const Wave& w, cudaStream_t s) {
    return stft_run(w, wcos, wsin, packed, n_fft, F, hop, out_format, sqrt_eps, out, T_max, workspace, ws_bytes,
                    path, s, &routes[0]);
  }, stream);
  if (rc == NNAB_OK) count_stft_routes(routes, g_stream_stft);
  return rc;
}

size_t nnab_filterbank_pool_workspace_bytes(int64_t A, int64_t T_max, int n_fft, int F, int hop, int n_fb,
                                            int path, int has_table) {
  const int64_t Lv = pool_clip_length(A, T_max, n_fft, hop);
  return Lv > 0 ? filterbank_ws_bytes(A, Lv, n_fft, F, hop, 0, n_fb, path, has_table) : 0;
}

int nnab_stft_filterbank_pool_forward(void* state, const nnab_stream_lane* lanes, const nnab_stream_lane* d_lanes,
                                      int64_t n_lanes, int64_t A, const void* chunk, int chunk_dtype, int64_t slots,
                                      int64_t n, int64_t chunk_pitch, const float* wcos, const float* wsin,
                                      const void* packed, int n_fft, int F, int hop, int center, int pad_mode,
                                      float sqrt_eps, float power, const float* fb, int n_fb, const void* fb_table,
                                      float* out, int64_t T_max, void* workspace, size_t ws_bytes, int path,
                                      void* stream) {
  PoolPlan pp;
  int rc = pool_plan(state, lanes, d_lanes, n_lanes, A, chunk, chunk_dtype, slots, n, chunk_pitch, n_fft, hop,
                     center ? n_fft / 2 : 0, pad_mode, T_max, &pp);
  if (rc) return rc;
  if (F <= 0 || (A > 0 && out == nullptr) || filterbank_args_ok(wcos, wsin, fb, n_fb)) return NNAB_EINVAL;
  int routes[2] = {-1, -1};
  rc = pool_forward(pp, chunk_dtype, n_lanes, out, n_fb, 1, [&](const Wave& w, cudaStream_t s) {
    return filterbank_run(w, wcos, wsin, packed, n_fft, F, hop, sqrt_eps, power, fb, n_fb, fb_table, out, T_max,
                          workspace, ws_bytes, path, s, &routes);
  }, stream);
  if (rc == NNAB_OK) count_stft_routes(routes, g_stream_stft);
  return rc;
}

size_t nnab_mfcc_pool_workspace_bytes(int64_t A, int64_t T_max, int n_fft, int F, int hop, int n_mels, int path,
                                      int has_table) {
  (void)has_table;
  const int64_t Lv = pool_clip_length(A, T_max, n_fft, hop);
  return Lv > 0 ? mfcc_ws_bytes(A, Lv, n_fft, F, hop, 0, n_mels, path) : 0;
}

int nnab_mfcc_pool_forward(void* state, const nnab_stream_lane* lanes, const nnab_stream_lane* d_lanes,
                           int64_t n_lanes, int64_t A, const void* chunk, int chunk_dtype, int64_t slots, int64_t n,
                           int64_t chunk_pitch, const float* wcos, const float* wsin, const void* packed, int n_fft,
                           int F, int hop, int center, int pad_mode, float sqrt_eps, float power,
                           const float* mel_basis, int n_mels, const void* fb_table, float amin, float ref,
                           float top_db, const float* dct, int n_mfcc, float* out, int64_t T_max, void* workspace,
                           size_t ws_bytes, int path, void* stream) {
  PoolPlan pp;
  int rc = pool_plan(state, lanes, d_lanes, n_lanes, A, chunk, chunk_dtype, slots, n, chunk_pitch, n_fft, hop,
                     center ? n_fft / 2 : 0, pad_mode, T_max, &pp);
  if (rc) return rc;
  // the top_db floor is a maximum over the whole clip: a stream cannot apply it frame by frame
  if (F <= 0 || (A > 0 && out == nullptr) || top_db >= 0.f ||
      mfcc_args_ok(wcos, wsin, mel_basis, n_mels, dct, n_mfcc, amin))
    return NNAB_EINVAL;
  int routes[2] = {-1, -1};
  rc = pool_forward(pp, chunk_dtype, n_lanes, out, n_mfcc, 1, [&](const Wave& w, cudaStream_t s) {
    return mfcc_run(w, wcos, wsin, packed, n_fft, F, hop, sqrt_eps, power, mel_basis, n_mels, fb_table, amin,
                    ref, top_db, dct, n_mfcc, out, T_max, workspace, ws_bytes, path, s, &routes);
  }, stream);
  if (rc == NNAB_OK) count_stft_routes(routes, g_stream_stft);
  return rc;
}

size_t nnab_cqt1992v2_pool_workspace_bytes(int64_t A, int64_t T_max, int width, int n_bins, int hop, int path) {
  const int64_t Lv = pool_clip_length(A, T_max, width, hop);
  return Lv > 0 ? nnab_cqt1992v2_workspace_bytes(A, Lv, width, n_bins, hop, 0, path) : 0;
}

int nnab_cqt1992v2_pool_forward(void* state, const nnab_stream_lane* lanes, const nnab_stream_lane* d_lanes,
                                int64_t n_lanes, int64_t A, const void* chunk, int chunk_dtype, int64_t slots,
                                int64_t n, int64_t chunk_pitch, const float* k_real, const float* k_imag,
                                const void* packed, const int32_t* h_k_begin, const int32_t* h_k_end, int n_bins,
                                int width, int hop, int center, int pad_mode, const float* scale, float scale_all,
                                int out_format, float sqrt_eps, float* out, int64_t T_max, void* workspace,
                                size_t ws_bytes, int path, void* stream) {
  PoolPlan pp;
  int rc = pool_plan(state, lanes, d_lanes, n_lanes, A, chunk, chunk_dtype, slots, n, chunk_pitch, width, hop,
                     center ? width / 2 : 0, pad_mode, T_max, &pp);
  if (rc) return rc;
  if (n_bins <= 0 || (A > 0 && out == nullptr) || cqt1992v2_args_ok(k_real, k_imag, out_format))
    return NNAB_EINVAL;
  int route = -1;
  rc = pool_forward(pp, chunk_dtype, n_lanes, out, n_bins, format_cols(out_format),
                      [&](const Wave& w, cudaStream_t s) {
    return cqt1992v2_run(w, k_real, k_imag, packed, h_k_begin, h_k_end, n_bins, width, hop, scale, scale_all,
                         out_format, sqrt_eps, out, T_max, workspace, ws_bytes, path, s, &route);
  }, stream);
  if (rc == NNAB_OK) count_cq1992_route(route, g_stream_cq1992);
  return rc;
}

// ------------------------------------------------------------ device pools ----
// T_cap: frame t is ready once thr(t) samples have arrived, so a stream one sample short of its first frame
// (thr - 1 samples: K - pad, and with reflect padding at least pad + 1) that takes `chunk` more and ends returns
// the most frames, ((thr - 1) + chunk + 2 pad - K) / hop + 1.  Later positions return at most
// ceil((chunk + pad) / hop), never more.
int64_t nnab_pool_frame_cap(int64_t chunk, int K, int hop, int pad, int pad_mode) {
  if (chunk < 1 || K < 2 || hop <= 0 || pad < 0 || 2 * pad > K) return 0;
  const int64_t need = (int64_t)K - pad;
  const int64_t thr = pad > 0 && pad_mode == NNAB_PAD_REFLECT && pad + 1 > need ? pad + 1 : need;
  return (thr - 1 + chunk + 2 * (int64_t)pad - K) / hop + 1;
}

int nnab_stft_pool_device_forward(void* state, int64_t* counters, const int32_t* lengths, const uint8_t* end,
                                  int32_t* errors, int64_t* error_info, int32_t* counts, nnab_stream_lane* d_lanes,
                                  const void* chunk, int chunk_dtype, int64_t slots, int64_t n, int64_t chunk_pitch,
                                  const float* wcos, const float* wsin, const void* packed, int n_fft, int F, int hop,
                                  int center, int pad_mode, int out_format, float sqrt_eps, float* out, int64_t T_max,
                                  void* workspace, size_t ws_bytes, int path, void* stream) {
  PoolPlan pp;
  int rc = device_pool_plan(state, counters, lengths, end, errors, error_info, counts, d_lanes, chunk, chunk_dtype,
                            slots, n, chunk_pitch, n_fft, hop, center ? n_fft / 2 : 0, pad_mode, T_max, out, &pp);
  if (rc) return rc;
  if (F <= 0 || stft_args_ok(wcos, wsin, out_format)) return NNAB_EINVAL;
  int routes[2] = {-1, -1};  // stays -1 when nothing was enqueued
  rc = device_pool_forward(pp, counters, lengths, end, errors, error_info, counts, chunk_dtype, n, out, F,
                           format_cols(out_format), [&](const Wave& w, cudaStream_t s) {
    return stft_run(w, wcos, wsin, packed, n_fft, F, hop, out_format, sqrt_eps, out, T_max, workspace, ws_bytes,
                    path, s, &routes[0]);
  }, stream);
  if (rc == NNAB_OK) count_stft_routes(routes, g_stream_stft);
  return rc;
}

int nnab_stft_filterbank_pool_device_forward(void* state, int64_t* counters, const int32_t* lengths,
                                             const uint8_t* end, int32_t* errors, int64_t* error_info,
                                             int32_t* counts, nnab_stream_lane* d_lanes, const void* chunk,
                                             int chunk_dtype, int64_t slots, int64_t n, int64_t chunk_pitch,
                                             const float* wcos, const float* wsin, const void* packed, int n_fft,
                                             int F, int hop, int center, int pad_mode, float sqrt_eps, float power,
                                             const float* fb, int n_fb, const void* fb_table, float* out,
                                             int64_t T_max, void* workspace, size_t ws_bytes, int path, void* stream) {
  PoolPlan pp;
  int rc = device_pool_plan(state, counters, lengths, end, errors, error_info, counts, d_lanes, chunk, chunk_dtype,
                            slots, n, chunk_pitch, n_fft, hop, center ? n_fft / 2 : 0, pad_mode, T_max, out, &pp);
  if (rc) return rc;
  if (F <= 0 || filterbank_args_ok(wcos, wsin, fb, n_fb)) return NNAB_EINVAL;
  int routes[2] = {-1, -1};
  rc = device_pool_forward(pp, counters, lengths, end, errors, error_info, counts, chunk_dtype, n, out, n_fb, 1,
                           [&](const Wave& w, cudaStream_t s) {
    return filterbank_run(w, wcos, wsin, packed, n_fft, F, hop, sqrt_eps, power, fb, n_fb, fb_table, out, T_max,
                          workspace, ws_bytes, path, s, &routes);
  }, stream);
  if (rc == NNAB_OK) count_stft_routes(routes, g_stream_stft);
  return rc;
}

int nnab_mfcc_pool_device_forward(void* state, int64_t* counters, const int32_t* lengths, const uint8_t* end,
                                  int32_t* errors, int64_t* error_info, int32_t* counts, nnab_stream_lane* d_lanes,
                                  const void* chunk, int chunk_dtype, int64_t slots, int64_t n, int64_t chunk_pitch,
                                  const float* wcos, const float* wsin, const void* packed, int n_fft, int F, int hop,
                                  int center, int pad_mode, float sqrt_eps, float power, const float* mel_basis,
                                  int n_mels, const void* fb_table, float amin, float ref, float top_db,
                                  const float* dct, int n_mfcc, float* out, int64_t T_max, void* workspace,
                                  size_t ws_bytes, int path, void* stream) {
  PoolPlan pp;
  int rc = device_pool_plan(state, counters, lengths, end, errors, error_info, counts, d_lanes, chunk, chunk_dtype,
                            slots, n, chunk_pitch, n_fft, hop, center ? n_fft / 2 : 0, pad_mode, T_max, out, &pp);
  if (rc) return rc;
  // the top_db floor is a maximum over the whole clip: a stream cannot apply it frame by frame
  if (F <= 0 || top_db >= 0.f || mfcc_args_ok(wcos, wsin, mel_basis, n_mels, dct, n_mfcc, amin)) return NNAB_EINVAL;
  int routes[2] = {-1, -1};
  rc = device_pool_forward(pp, counters, lengths, end, errors, error_info, counts, chunk_dtype, n, out, n_mfcc, 1,
                           [&](const Wave& w, cudaStream_t s) {
    return mfcc_run(w, wcos, wsin, packed, n_fft, F, hop, sqrt_eps, power, mel_basis, n_mels, fb_table, amin,
                    ref, top_db, dct, n_mfcc, out, T_max, workspace, ws_bytes, path, s, &routes);
  }, stream);
  if (rc == NNAB_OK) count_stft_routes(routes, g_stream_stft);
  return rc;
}

int nnab_cqt1992v2_pool_device_forward(void* state, int64_t* counters, const int32_t* lengths, const uint8_t* end,
                                       int32_t* errors, int64_t* error_info, int32_t* counts,
                                       nnab_stream_lane* d_lanes, const void* chunk, int chunk_dtype, int64_t slots,
                                       int64_t n, int64_t chunk_pitch, const float* k_real, const float* k_imag,
                                       const void* packed, const int32_t* h_k_begin, const int32_t* h_k_end,
                                       int n_bins, int width, int hop, int center, int pad_mode, const float* scale,
                                       float scale_all, int out_format, float sqrt_eps, float* out, int64_t T_max,
                                       void* workspace, size_t ws_bytes, int path, void* stream) {
  PoolPlan pp;
  int rc = device_pool_plan(state, counters, lengths, end, errors, error_info, counts, d_lanes, chunk, chunk_dtype,
                            slots, n, chunk_pitch, width, hop, center ? width / 2 : 0, pad_mode, T_max, out, &pp);
  if (rc) return rc;
  if (n_bins <= 0 || cqt1992v2_args_ok(k_real, k_imag, out_format)) return NNAB_EINVAL;
  int route = -1;
  rc = device_pool_forward(pp, counters, lengths, end, errors, error_info, counts, chunk_dtype, n, out, n_bins,
                           format_cols(out_format), [&](const Wave& w, cudaStream_t s) {
    return cqt1992v2_run(w, k_real, k_imag, packed, h_k_begin, h_k_end, n_bins, width, hop, scale, scale_all,
                         out_format, sqrt_eps, out, T_max, workspace, ws_bytes, path, s, &route);
  }, stream);
  if (rc == NNAB_OK) count_cq1992_route(route, g_stream_cq1992);
  return rc;
}

// ---- PCEN (pcen_kernels.cu) ----
static bool pcen_shape_ok(const float* s, const float* gain, const float* bias, const float* power,
                          int param_stride, float eps, int64_t B, int C, int64_t T) {
  return s != nullptr && gain != nullptr && bias != nullptr && power != nullptr &&
         (param_stride == 0 || param_stride == 1) && eps > 0.f && eps < INFINITY && B >= 0 && C >= 1 && T >= 0 &&
         pcen_blocks(B * (int64_t)C) < (int64_t)INT32_MAX;
}

size_t nnab_pcen_workspace_bytes(int64_t B, int C) {
  return (B < 0 || C < 1) ? 0 : 4 * (size_t)B * (size_t)C * sizeof(float);
}

int nnab_pcen_forward(const float* E, int64_t B, int C, int64_t T, const float* s, const float* gain,
                      const float* bias, const float* power, int param_stride, float eps, float* P, float* M,
                      float* state, uint8_t* primed, int64_t slots, const int32_t* row_slot, const int32_t* counts,
                      void* stream) {
  // an empty spectrogram may come without storage: its pointers are only checked when there are frames
  if (((E == nullptr || P == nullptr) && B * T > 0) ||
      !pcen_shape_ok(s, gain, bias, power, param_stride, eps, B, C, T))
    return NNAB_EINVAL;
  if ((state == nullptr) != (primed == nullptr)) return NNAB_EINVAL;
  if (state == nullptr && (row_slot != nullptr || counts != nullptr)) return NNAB_EINVAL;  // stream-only arguments
  if (state != nullptr && (M != nullptr || slots < 1 || (row_slot == nullptr && B > slots))) return NNAB_EINVAL;
  const int rc = check_arch();
  if (rc) return rc;
  if (B == 0 || T == 0) return NNAB_OK;
  return pcen_forward(E, B, C, T, PcenArgs{s, gain, bias, power, param_stride, eps}, P, M,
                      PcenStream{state, primed, slots, row_slot, counts}, (cudaStream_t)stream);
}

int nnab_pcen_backward(const float* E, const float* M, const float* grad_P, int64_t B, int C, int64_t T,
                       const float* s, const float* gain, const float* bias, const float* power, int param_stride,
                       float eps, float* grad_E, float* grad_params, void* workspace, size_t ws_bytes, void* stream) {
  if (((E == nullptr || M == nullptr || grad_P == nullptr) && B * T > 0) ||
      !pcen_shape_ok(s, gain, bias, power, param_stride, eps, B, C, T))
    return NNAB_EINVAL;
  const int rc = check_arch();
  if (rc) return rc;
  const size_t ws_need = grad_params != nullptr ? nnab_pcen_workspace_bytes(B, C) : 0;
  if (ws_need > 0 && (workspace == nullptr || ws_bytes < ws_need)) return NNAB_EWORKSPACE;
  if (B == 0 || T == 0) {  // no frames: grad_E is empty and every parameter gradient is zero
    if (grad_params != nullptr)
      NNAB_CUDA_TRY(cudaMemsetAsync(grad_params, 0, 4 * (size_t)(param_stride ? C : 1) * sizeof(float),
                                    (cudaStream_t)stream));
    return NNAB_OK;
  }
  if (grad_E == nullptr && grad_params == nullptr) return NNAB_OK;
  return pcen_backward(E, M, grad_P, B, C, T, PcenArgs{s, gain, bias, power, param_stride, eps}, grad_E, grad_params,
                       static_cast<float*>(workspace), (cudaStream_t)stream);
}

int nnab_pcen_reset(uint8_t* primed, const uint8_t* mask, int64_t slots, int C, void* stream) {
  if (primed == nullptr || slots < 1 || C < 1) return NNAB_EINVAL;
  const int rc = check_arch();
  if (rc) return rc;
  return pcen_reset(primed, mask, slots, C, (cudaStream_t)stream);
}

}  // extern "C"
