// Host-side pieces shared by the tensor-core translation units (tc_kernels.cu, tcb_kernels.cu).
#pragma once

#include <cuda.h>
#include <stdint.h>

#include "common.cuh"

namespace nnab {

constexpr int TC_BM = 128;
constexpr int TC_THREADS = 256;

static inline int round_up_i(int v, int a) { return (v + a - 1) / a * a; }

// geometry of the split / padded signal workspace (tc_kernels.cu)
struct SplitGeom {
  int64_t t_slots;       // virtual frames per clip
  int64_t nv;            // virtual frames in the batch
  int64_t rows;          // rows of the (rows x hop) view incl. K overhang
  int64_t plane_stride;  // elements per plane
};
SplitGeom split_geom(int64_t B, int64_t L, int K, int hop, int pad);
int num_phases(int hop);

// bf16 3-D tensor map {d0 (contiguous), d1, d2}, box {box0, box1, 1}, swizzle by bk (64 -> 128B)
int encode_3d(CUtensorMap* map, void* base, uint64_t d0, uint64_t d1, uint64_t d2,
              uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t box0, uint32_t box1, int bk);

int encode_4d(CUtensorMap* map, void* base, const uint64_t dims[4], const uint64_t strides[3],
              const uint32_t box[3]);
size_t tc_packed_bytes(int F, int K);
int tc_pack_basis_varn(const float* w_re, const float* w_im, int F, int K, void* packed,
                       cudaStream_t stream);

// layout of a packed basis, keyed by its device pointer
enum { PACK_DENSE = 0, PACK_VARN = 2, PACK_BLOCK = 4 };
int packed_kind(const void* packed);
void mark_packed(const void* packed, int kind);

// block-partial ("sliding") STFT kernel (tcb_kernels.cu)
int tc_pack_basis_block(int n_fft, int hop, void* packed, cudaStream_t stream);
size_t tc_packed_block_bytes(int n_fft, int hop);
bool tc_block_shape_ok(int n_fft, int hop);
int launch_framed_tc_block(const FramedProblem& q, const void* packed, void* workspace,
                           size_t ws_bytes, cudaStream_t stream);

// tall-A kernel for long nested banks (tct_kernels.cu); NNAB_EUNSUPPORTED = not applicable, nothing enqueued
int launch_framed_tc_tall(const FramedProblem& q, const void* packed, void* workspace, size_t ws_bytes,
                          cudaStream_t stream);

// FIR decimator stage with banded taps (tct_kernels.cu); NNAB_EUNSUPPORTED = geometry not eligible
int launch_fir_stage_tc(const void* src_planes, int64_t B, int64_t src_len, int64_t src_pitch,
                        int64_t src_plane_stride, int src_pad, const void* fir_packed,
                        const float* fir, int taps, const DecimParams& dec, cudaStream_t stream);

// octave CQT on shared level planes: resident bank, tall A blocks, frame phases (tct_kernels.cu)
int launch_octave_tc(const FramedProblem& q, const void* packed, cudaStream_t stream);
int tc_tile_n(int F);

}  // namespace nnab
