// PTX wrappers for the tensor-core kernels (sm_90a): TMA, mbarrier, wgmma, and the shared-memory
// accumulator tile their epilogues read.  Shared by tc_kernels.cu, tcb_kernels.cu and tct_kernels.cu.
//
// Common shape of those kernels: 288 threads = two consumer warpgroups (warps 0-7) and one TMA producer
// warp (warp 8).  A 128-row tile of the framed GEMM is two m64 wgmma halves, one per consumer warpgroup,
// accumulated in registers; when a tile's K range is done both warpgroups store their fragments into the
// accumulator tile, and the consumer warps run the epilogue from there, one tile row per thread.
#pragma once

#include <cuda.h>
#include <stdint.h>

#include "wgmma_bf16.cuh"

namespace nnab {

constexpr int TC_CONSUMER_THREADS = 256;                     // warps 0-7: two wgmma warpgroups
constexpr int TC_KERNEL_THREADS = TC_CONSUMER_THREADS + 32;  // + warp 8: TMA producer
constexpr int TC_PRODUCER_WARP = 8;

// ---------------------------------------------------------------------------
// mbarrier / TMA
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a descriptor / barrier bug must trap, never hang the GPU.  (No printf here: a call in a
// kernel that keeps wgmma accumulators in registers makes ptxas serialise every wgmma.)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  unsigned long long t0 = 0;
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0xFFFu) == 0) {
      unsigned long long now;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000ull) __trap();  // 4 s
    }
  }
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// generic-proxy accesses of shared memory before async-proxy (TMA) writes of the same bytes
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
// barrier over the 256 consumer threads only (the producer warp keeps streaming)
__device__ __forceinline__ void consumer_sync() {
  asm volatile("bar.sync 1, %0;" ::"n"(TC_CONSUMER_THREADS) : "memory");
}

// ---------------------------------------------------------------------------
// wgmma
// ---------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_wait_all() {
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}
// at most `PENDING` committed groups of this warpgroup still in flight
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory");
}

// K-major SWIZZLE_128B shared-memory matrix descriptor (64 bf16 = 128 B per row, 8-row atoms):
//   [0,14) start >> 4 | [16,30) LBO >> 4 (unused when swizzled) | [32,46) SBO >> 4 = 1024 B | [62,64) 1
// The low word is (addr >> 4) | 1 << 16: moving along K (+32 B per K16 slice) or down rows (+128 B per
// row) is an add of the low word.  The swizzle is a function of the address bits, so an operand may
// start at any 128-byte row of a TMA-written block (tc_probe.cu checks this on the device).
__device__ __forceinline__ uint32_t wg_desc_lo(uint32_t saddr) { return ((saddr & 0x3FFFFu) >> 4) | (1u << 16); }
__device__ __forceinline__ uint32_t wg_desc_hi() { return (1024u >> 4) | (1u << 30); }
// K-major SWIZZLE_64B (32 bf16 = 64 B per row): SBO = 8 rows = 512 B, layout type [62,64) 2.  The low word
// is the same; a K16 slice is still +32 B.  An operand starts at a 512-byte boundary (one swizzle atom).
__device__ __forceinline__ uint32_t wg_desc_hi_sw64() { return (512u >> 4) | (2u << 30); }
__device__ __forceinline__ uint64_t desc64(uint32_t lo, uint32_t hi) {
  uint64_t d;
  asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "r"(lo), "r"(hi));
  return d;
}

// One K block (BK = 64: four K16 slices, SWIZZLE_128B; BK = 32: two, SWIZZLE_64B) of the 3-term bf16
// split, x*w ~= xlo*whi + xhi*wlo + xhi*whi, for this warpgroup's 64 rows: A (hi, lo planes) x B (hi, lo
// planes) -> d (N / 2 registers).  Arguments are the low descriptor words of the four operand blocks.
template <int N, int BK = 64>
__device__ __forceinline__ void wg_kblock_split3_n(float* d, uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                                   uint32_t b_lo, bool first_accumulates) {
  static_assert(BK == 64 || BK == 32, "K block is one 128-byte or 64-byte swizzled row");
  const uint32_t hi = (BK == 64) ? wg_desc_hi() : wg_desc_hi_sw64();
#pragma unroll
  for (int k = 0; k < BK / 16; ++k) {
    const uint32_t o = 2u * k;
    Wgmma<N>::mma(d, desc64(a_lo + o, hi), desc64(b_hi + o, hi), (k == 0 && !first_accumulates) ? 0u : 1u);
    Wgmma<N>::mma(d, desc64(a_hi + o, hi), desc64(b_lo + o, hi), 1u);
    Wgmma<N>::mma(d, desc64(a_hi + o, hi), desc64(b_hi + o, hi), 1u);
  }
}

// The 2-term form for an A operand that is exactly bf16 (a bf16 waveform: xlo == 0), xhi*wlo + xhi*whi.
// It issues the last two wgmmas of wg_kblock_split3_n in the same order, so every accumulator gets what
// the 3-term form gives on a zero lo plane (there, d + 0 = d), up to the sign of a zero.
template <int N, int BK = 64>
__device__ __forceinline__ void wg_kblock_split2_n(float* d, uint32_t a_hi, uint32_t b_hi, uint32_t b_lo,
                                                   bool first_accumulates) {
  static_assert(BK == 64 || BK == 32, "K block is one 128-byte or 64-byte swizzled row");
  const uint32_t hi = (BK == 64) ? wg_desc_hi() : wg_desc_hi_sw64();
#pragma unroll
  for (int k = 0; k < BK / 16; ++k) {
    const uint32_t o = 2u * k;
    Wgmma<N>::mma(d, desc64(a_hi + o, hi), desc64(b_lo + o, hi), (k == 0 && !first_accumulates) ? 0u : 1u);
    Wgmma<N>::mma(d, desc64(a_hi + o, hi), desc64(b_hi + o, hi), 1u);
  }
}

// the same with N chosen at run time (a multiple of 16, <= NMAX); d holds NMAX / 2 registers
template <int NMAX>
__device__ __forceinline__ void wg_kblock_split3(int n, float* d, uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                                 uint32_t b_lo, bool first_accumulates) {
  switch (n) {
#define NNAB_WG_CASE(N)                                                                   \
  case N:                                                                                 \
    if constexpr (N <= NMAX) wg_kblock_split3_n<N>(d, a_hi, a_lo, b_hi, b_lo, first_accumulates); \
    break;
    NNAB_WG_CASE(16) NNAB_WG_CASE(32) NNAB_WG_CASE(48) NNAB_WG_CASE(64)
    NNAB_WG_CASE(80) NNAB_WG_CASE(96) NNAB_WG_CASE(112) NNAB_WG_CASE(128)
    NNAB_WG_CASE(144) NNAB_WG_CASE(160) NNAB_WG_CASE(176) NNAB_WG_CASE(192)
    NNAB_WG_CASE(208) NNAB_WG_CASE(224) NNAB_WG_CASE(240) NNAB_WG_CASE(256)
#undef NNAB_WG_CASE
    default: break;
  }
}

// ---------------------------------------------------------------------------
// Accumulator tile: 128 fp32 rows of `stride` bytes (a multiple of 128) at the 1024-aligned start of
// dynamic shared memory.  The 16-byte chunk c of row r is stored at chunk position c ^ (r & 7): a warp
// reading the same chunk of 32 consecutive rows, and a warpgroup storing its wgmma fragments, spread over
// all banks.
//
// An accumulator address packs: bits [0,16) column, [16,24) row read by lane 0, [24,28) stride / 128 B.
// acc_ld8 / acc_ld32 read 8 / 32 consecutive columns of row (lane-0 row + lane) into every lane.
// ---------------------------------------------------------------------------
extern __shared__ __align__(1024) uint8_t nnab_dyn_smem[];

__device__ __forceinline__ uint32_t acc_tile_base() { return (smem_u32(nnab_dyn_smem) + 1023u) & ~1023u; }
// address of column 0, row 0 of a tile whose rows are `cols` fp32 wide (rounded up to 32 columns)
__device__ __forceinline__ uint32_t acc_tile(int cols) { return (uint32_t)((cols + 31) >> 5) << 24; }
__device__ __forceinline__ uint32_t acc_row(uint32_t row) { return row << 16; }

__device__ __forceinline__ uint32_t acc_chunk_smem(uint32_t taddr, uint32_t row) {
  const uint32_t col = taddr & 0xFFFFu;
  const uint32_t chunk = col >> 2;
  const uint32_t pos = (chunk & ~7u) | ((chunk ^ row) & 7u);
  return acc_tile_base() + row * ((taddr >> 24) << 7) + pos * 16u + (col & 3u) * 4u;
}
__device__ __forceinline__ void acc_ld4(uint32_t taddr, uint32_t row, uint32_t* v) {
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3])
               : "r"(acc_chunk_smem(taddr, row))
               : "memory");
}
__device__ __forceinline__ void acc_st4(uint32_t taddr, uint32_t row, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(acc_chunk_smem(taddr, row)), "f"(a), "f"(b),
               "f"(c), "f"(d)
               : "memory");
}
__device__ __forceinline__ void acc_ld8(uint32_t taddr, uint32_t (&v)[8]) {
  const uint32_t row = ((taddr >> 16) & 0xFFu) + (threadIdx.x & 31u);
  acc_ld4(taddr, row, v);
  acc_ld4(taddr + 4u, row, v + 4);
}
__device__ __forceinline__ void acc_ld32(uint32_t taddr, uint32_t (&v)[32]) {
  const uint32_t row = ((taddr >> 16) & 0xFFu) + (threadIdx.x & 31u);
#pragma unroll
  for (int i = 0; i < 8; ++i) acc_ld4(taddr + 4u * i, row, v + 4 * i);
}

// Store this warpgroup's accumulator fragment (rows [row0, row0 + 64), columns [0, n)) into the tile.
template <int NMAX>
__device__ __forceinline__ void acc_store(uint32_t tile, const float* d, int n, int row0) {
  const uint32_t t = threadIdx.x & 127u;
  const uint32_t r = (uint32_t)row0 + (t >> 5) * 16u + ((t & 31u) >> 2);
  const uint32_t c = (t & 3u) * 2u;
#pragma unroll
  for (int j = 0; j < NMAX / 8; ++j) {
    if (8 * j < n) {
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(acc_chunk_smem(tile + 8u * j + c, r)),
                   "f"(d[4 * j]), "f"(d[4 * j + 1])
                   : "memory");
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(acc_chunk_smem(tile + 8u * j + c, r + 8u)),
                   "f"(d[4 * j + 2]), "f"(d[4 * j + 3])
                   : "memory");
    }
  }
}

}  // namespace nnab
