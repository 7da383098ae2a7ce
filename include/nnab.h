/*
 * nnab.h — C ABI of the nnaudio-b200 hot path (libnnab.so).
 *
 * The reference (KinWaiCheuk/nnAudio v0.3.3) is pure Python/PyTorch and has no
 * FFI of its own; its hot path is the body of each module's forward():
 * reflect/constant centre padding, conv1d(x, basis, stride=hop) framing +
 * contraction, and the element-wise / filterbank / dB / DCT tail.  Each entry
 * point below replaces exactly one such forward body (file:line cited per
 * function, paths relative to Installation/nnAudio/) and is what a ctypes /
 * cffi binding inside the reference would call (see INTEGRATION.md).
 *
 * Conventions (all entry points):
 *   - plain C types only; every data pointer is a DEVICE pointer owned by the
 *     caller unless the name starts with h_ (host memory);
 *   - inputs are the reference's own fp32 buffers, in the reference's own
 *     layouts (row-major, last dim contiguous); outputs are freshly written
 *     contiguous fp32 tensors in the reference's output layout;
 *   - work is enqueued on `stream` (a cudaStream_t passed as void*); the call
 *     never synchronises, never allocates device memory and never throws;
 *   - return 0 on success or a negative nnab_status; nnab_strerror() names it;
 *   - `workspace` is caller-provided scratch of at least the number of bytes
 *     the matching nnab_*_workspace_bytes() query returns (may be NULL iff
 *     that query returns 0);
 *   - `path` selects the kernel family: NNAB_PATH_AUTO picks the tensor-core
 *     (wgmma/TMA) kernels when shape/alignment allow and the packed basis is
 *     supplied, otherwise the generic SIMT kernel.  Both are sm_90a CUDA; there
 *     is no CPU fallback.  NNAB_PATH_TCGEN05 forces the tensor-core kernels.
 */
#ifndef NNAB_H_
#define NNAB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* every entry point below is exported; everything else in the library is hidden */
#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

#define NNAB_ABI_VERSION 1

typedef enum nnab_status {
  NNAB_OK = 0,
  NNAB_EINVAL = -1,     /* bad argument / shape mismatch                      */
  NNAB_EALIGN = -2,     /* forced tensor-core path, alignment rules not met   */
  NNAB_EARCH = -3,      /* device is not sm_90 (compute capability 9.0)       */
  NNAB_ECUDA = -4,      /* a CUDA runtime / driver call failed                */
  NNAB_EWORKSPACE = -5, /* workspace NULL or too small                        */
  NNAB_EUNSUPPORTED = -6
} nnab_status;

/* centre padding mode (stft.py:278-289, cqt.py:740-746) */
#define NNAB_PAD_REFLECT 0
#define NNAB_PAD_CONSTANT 1

/* output formats */
#define NNAB_FMT_MAGNITUDE 0   /* (B, F, T)     sqrt(re^2 + im^2 [+ eps])            */
#define NNAB_FMT_COMPLEX 1     /* (B, F, T, 2)  (re, im)                             */
#define NNAB_FMT_PHASE_ANGLE 2 /* (B, F, T)     atan2(im + 0.0, re)   STFT 'Phase'   */
#define NNAB_FMT_PHASE_UNIT 3  /* (B, F, T, 2)  (cos, sin)(atan2(im, re)) CQT 'Phase'*/

/* kernel family */
#define NNAB_PATH_AUTO 0
#define NNAB_PATH_SIMT 1
#define NNAB_PATH_TCGEN05 2

/* Sample type of the waveform `x` of the *_forward_ex entry points.  Everything else (bases, filterbanks,
 * outputs) stays fp32, and the result is the fp32 transform of the given samples: the tensor-core
 * pre-pass converts each sample to fp32 exactly before splitting it.  Plans that would read `x` as
 * fp32 directly (the SIMT kernels, the per-octave CQT pyramid) return NNAB_EUNSUPPORTED for a 16-bit
 * `x` before anything is enqueued; the caller may then upcast and call again. */
#define NNAB_DTYPE_F32 0
#define NNAB_DTYPE_BF16 1
#define NNAB_DTYPE_F16 2

int nnab_abi_version(void);
const char* nnab_strerror(int status);
/* Last CUDA error string recorded by a call that returned NNAB_ECUDA (thread local). */
const char* nnab_last_cuda_error(void);

/* ------------------------------------------------------------------------- *
 * Basis packing for the tensor-core path.
 *
 * Splits the fp32 basis pair (re rows, im rows), each (F, K) row-major, into
 * bf16 hi/lo planes (x = hi + lo to ~2^-17) laid out for TMA/wgmma:
 *   packed[plane][tile*BN + part*BN/2 + j][k]   plane 0 = hi, 1 = lo
 *   part 0 = re rows, part 1 = NEGATED im rows, j < BN/2 bins per tile
 * with K padded to a multiple of 64 and bins zero-padded to a multiple of BN/2.
 * BN = nnab_pack_tile_n(F) is chosen per basis to minimise padded columns (208
 * for F = 1025; <= 256).  Negation folds the reference's minus signs
 * (stft.py:308-311 `-spec_imag`, cqt.py:750 `-conv1d(...)`) into the basis.
 * ------------------------------------------------------------------------- */
int nnab_pack_tile_n(int F);
size_t nnab_packed_basis_bytes(int F, int K);
int nnab_pack_basis(const float* w_re, const float* w_im, int F, int K,
                    void* packed, void* stream);
/* Same buffer size, explicit layout request:
 *   NNAB_LAYOUT_DENSE (0)   the layout above
 *   NNAB_LAYOUT_GROUPS (3)  8-bin (re | im) row groups for long nested banks (F <= 128, CQT1992v2): the
 *                           per-K-block-width and tall-A kernels skip the zeros of the shorter wavelets.
 * The forward entry points recognise the layout of the buffer they are given. */
#define NNAB_LAYOUT_DENSE 0
#define NNAB_LAYOUT_GROUPS 3
int nnab_pack_basis_ex(const float* w_re, const float* w_im, int F, int K, int layout,
                       void* packed, void* stream);

/* Block-partial ("sliding") layout for the STFT family: periodic Hann window of length n_fft,
 * integer bins (freq_scale='no', F = n_fft/2 + 1) and hop = n_fft/R with R = 2 or 4, hop % 64 == 0
 * -- the reference's defaults (stft.py:177-178, utils.py:379-384).  The contraction then runs once
 * per hop-sized block against the UN-windowed basis (K = hop instead of n_fft: R x fewer MMA flops);
 * the window is a 3-tap filter along the bin axis and the frame sum a combination of R consecutive
 * block rows, both in the kernel's epilogue.  The packed rows are generated analytically (float64),
 * so the CALLER vouches that its wcos/wsin buffers are exactly that transform
 * (nnaudio_b200/features/_common.py:is_hann_dft checks the tensors).  `packed` needs
 * nnab_packed_block_bytes(n_fft, hop) bytes; the forward entry points recognise the layout.
 * nnab_block_layout_ok() is host-only: 1 when (n_fft, hop) is eligible. */
int nnab_block_layout_ok(int n_fft, int hop);

/* Stream-ordered 32-bit store / cyclic >= wait on a device address (may be peer-mapped): front-end
 * memory operations (cuStreamWriteValue32 / cuStreamWaitValue32), no kernel, no SM.  The multi-GPU
 * gather uses them for its slot handshakes (nnaudio_b200/parallel.py). */
int nnab_stream_write_value32(void* stream, void* addr, uint32_t value);
int nnab_stream_wait_value32_geq(void* stream, void* addr, uint32_t value);
size_t nnab_packed_block_bytes(int n_fft, int hop);
int nnab_pack_basis_block(int n_fft, int hop, void* packed, void* stream);

/* ------------------------------------------------------------------------- *
 * STFT.forward — features/stft.py:256-316.
 *   x        (B, L) rows with pitch x_pitch floats
 *   wcos/wsin (F, n_fft) = the module's `wcos` / `wsin` buffers (window applied)
 *   out      Magnitude/Phase: (B, F, T); Complex: (B, F, T, 2) = (real, -imag)
 *   T must equal (L + 2*pad - n_fft)/hop + 1, pad = center ? n_fft/2 : 0
 *   sqrt_eps = 1e-8 iff the module is trainable (stft.py:301-304), else 0
 * ------------------------------------------------------------------------- */
size_t nnab_stft_workspace_bytes(int64_t B, int64_t L, int n_fft, int F, int hop,
                                 int center, int path);
int nnab_stft_forward(const float* x, int64_t B, int64_t L, int64_t x_pitch,
                      const float* wcos, const float* wsin, const void* packed,
                      int n_fft, int F, int hop, int center, int pad_mode,
                      int out_format, float sqrt_eps, float* out, int64_t T,
                      void* workspace, size_t ws_bytes, int path, void* stream);
/* The same for a waveform of sample type x_dtype (NNAB_DTYPE_*); x_pitch stays in samples.
 * nnab_stft_forward is this call with NNAB_DTYPE_F32; so are the other *_forward / *_forward_ex pairs. */
int nnab_stft_forward_ex(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch,
                         const float* wcos, const float* wsin, const void* packed,
                         int n_fft, int F, int hop, int center, int pad_mode,
                         int out_format, float sqrt_eps, float* out, int64_t T,
                         void* workspace, size_t ws_bytes, int path, void* stream);

/* ------------------------------------------------------------------------- *
 * Banded filterbank table (tensor-core path): for every FFT bin the (at most two)
 * non-zero weights of the (n_fb, F) filterbank.  Mel banks are banded like that;
 * for denser banks (gammatone) *h_max_nnz > 2 and the forward calls must be
 * given fb_table = NULL (they then run the un-fused filterbank GEMM).
 * Init-time helper: this call synchronises `stream` to return *h_max_nnz.
 * ------------------------------------------------------------------------- */
size_t nnab_filterbank_table_bytes(int F);
int nnab_build_filterbank_table(const float* fb, int n_fb, int F, void* table,
                                int* h_max_nnz, void* stream);
/* 1 when a forward call given this table (built above), this packed basis and n_fft sums the bank in the
 * contraction's epilogue, 0 when it runs the un-fused filterbank: pass the result as `has_table` to the workspace
 * queries.  The epilogue adds one fp32 atomic partial sum per N tile a filter's bins meet; on a dense basis the
 * table is used only when that is at most two for every filter, so that the sum does not depend on the order they
 * land in, and only for n_fft < 8192: a longer basis needs the split-K accumulation only the un-fused power
 * spectrogram has. */
int nnab_filterbank_table_fuses(const void* table, const void* packed, int n_fft);

/* ------------------------------------------------------------------------- *
 * MelSpectrogram.forward / Gammatonegram.forward — features/mel.py:171-189,
 * features/gammatone.py:171-189:  out = fb @ (|STFT(x)| ** power).
 *   fb (n_fb, F) = `mel_basis` or `gammatone_basis`;  out (B, n_fb, T)
 *   fb_table: table from nnab_build_filterbank_table (max_nnz <= 2) or NULL.
 *     With a table and the tensor-core path the filterbank is applied in the
 *     contraction kernel's epilogue (no (B,F,T) intermediate in HBM).
 * ------------------------------------------------------------------------- */
size_t nnab_filterbank_workspace_bytes(int64_t B, int64_t L, int n_fft, int F, int hop,
                                       int center, int n_fb, int path, int has_table);
int nnab_stft_filterbank_forward(const float* x, int64_t B, int64_t L, int64_t x_pitch,
                                 const float* wcos, const float* wsin, const void* packed,
                                 int n_fft, int F, int hop, int center, int pad_mode,
                                 float sqrt_eps, float power, const float* fb, int n_fb,
                                 const void* fb_table, float* out, int64_t T,
                                 void* workspace, size_t ws_bytes, int path, void* stream);
int nnab_stft_filterbank_forward_ex(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch,
                                    const float* wcos, const float* wsin, const void* packed,
                                    int n_fft, int F, int hop, int center, int pad_mode,
                                    float sqrt_eps, float power, const float* fb, int n_fb,
                                    const void* fb_table, float* out, int64_t T,
                                    void* workspace, size_t ws_bytes, int path, void* stream);

/* ------------------------------------------------------------------------- *
 * MFCC.forward — features/mel.py:309-326 (= mel -> _power_to_db :263-279 ->
 * _dct(norm='ortho') :281-307 -> [:, :n_mfcc]).
 *   top_db < 0 means None;  dct (n_mfcc, n_mels) fp32 orthonormal DCT-II rows;
 *   out (B, n_mfcc, T)
 * ------------------------------------------------------------------------- */
size_t nnab_mfcc_workspace_bytes(int64_t B, int64_t L, int n_fft, int F, int hop,
                                 int center, int n_mels, int path, int has_table);
int nnab_mfcc_forward(const float* x, int64_t B, int64_t L, int64_t x_pitch,
                      const float* wcos, const float* wsin, const void* packed,
                      int n_fft, int F, int hop, int center, int pad_mode,
                      float sqrt_eps, float power, const float* mel_basis, int n_mels,
                      const void* fb_table, float amin, float ref, float top_db,
                      const float* dct, int n_mfcc, float* out, int64_t T,
                      void* workspace, size_t ws_bytes, int path, void* stream);
int nnab_mfcc_forward_ex(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch,
                         const float* wcos, const float* wsin, const void* packed,
                         int n_fft, int F, int hop, int center, int pad_mode,
                         float sqrt_eps, float power, const float* mel_basis, int n_mels,
                         const void* fb_table, float amin, float ref, float top_db,
                         const float* dct, int n_mfcc, float* out, int64_t T,
                         void* workspace, size_t ws_bytes, int path, void* stream);

/* ------------------------------------------------------------------------- *
 * CQT1992v2.forward — features/cqt.py:712-780.
 *   k_real/k_imag (n_bins, width) = `cqt_kernels_real/imag` buffers
 *   h_k_begin/h_k_end: HOST int32[n_bins], the non-zero tap support
 *     [begin, end) of every bin (NULL = treat the bank as dense)
 *   scale: DEVICE fp32[n_bins] per-bin factor (sqrt(lenghts) for 'librosa') or
 *     NULL; scale_all: scalar factor (2 for 'wrap', else 1)
 *   out_format: MAGNITUDE, COMPLEX (real, imag) or PHASE_UNIT (cos, sin)
 * ------------------------------------------------------------------------- */
size_t nnab_cqt1992v2_workspace_bytes(int64_t B, int64_t L, int width, int n_bins, int hop,
                                      int center, int path);
int nnab_cqt1992v2_forward(const float* x, int64_t B, int64_t L, int64_t x_pitch,
                           const float* k_real, const float* k_imag, const void* packed,
                           const int32_t* h_k_begin, const int32_t* h_k_end,
                           int n_bins, int width, int hop, int center, int pad_mode,
                           const float* scale, float scale_all, int out_format,
                           float sqrt_eps, float* out, int64_t T,
                           void* workspace, size_t ws_bytes, int path, void* stream);
int nnab_cqt1992v2_forward_ex(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch,
                              const float* k_real, const float* k_imag, const void* packed,
                              const int32_t* h_k_begin, const int32_t* h_k_end,
                              int n_bins, int width, int hop, int center, int pad_mode,
                              const float* scale, float scale_all, int out_format,
                              float sqrt_eps, float* out, int64_t T,
                              void* workspace, size_t ws_bytes, int path, void* stream);

/* ------------------------------------------------------------------------- *
 * CQT2010v2.forward / VQT.forward — features/cqt.py:1070-1139,
 * features/vqt.py:143-215 (+ utils.py:73-124 downsampling, :498-521
 * get_cqt_complex with its reflect -> zero-padding fallback).
 *   h_k_real/h_k_imag: HOST arrays of n_octaves DEVICE pointers, octave 0 = top;
 *     bank i is (n_filters, h_widths[i]) fp32 (CQT2010v2 passes the same bank
 *     n_octaves times)
 *   lowpass (256) = `lowpass_filter`; early_filter (256) or NULL with
 *     early_factor (1 = inactive) = `early_downsample_filter`
 *   hop = the module's hop_length AFTER early downsampling
 *   scale: DEVICE fp32[n_bins] = downsample_factor * sqrt(lenghts) etc.
 *   out (B, n_bins, T[, 2]);  T = floor(L_early / hop) + 1 for every octave,
 *     otherwise NNAB_EINVAL (the reference's torch.cat would fail)
 * ------------------------------------------------------------------------- */
/* Packed (bf16 hi/lo, banded-Toeplitz) form of a 256-tap decimation FIR for the
 * tensor-core pyramid: lowpass_filter with dec = 2, early_downsample_filter with
 * dec = early_factor.  Init-time, cached by the caller. */
size_t nnab_packed_fir_bytes(int taps, int dec);
int nnab_pack_fir(const float* fir, int taps, int dec, void* packed, void* stream);

/* Host only (tests / tooling): the K-block plan of the per-block-width kernel
 * (order[i] = 64-sample K block, groups[i] = 8-bin groups it reaches, widest first;
 * chunk_begin[0..n_chunks] = split-K chunks of equal modelled cost).  Arrays: 512 / 512 / 17 ints. */
int nnab_debug_varn_plan(const int32_t* h_k_begin, const int32_t* h_k_end, int n_bins, int width,
                         int want_chunks, int32_t* order, int32_t* groups, int32_t* chunk_begin,
                         int32_t* n_blocks, int32_t* n_chunks);

/* One decimating-FIR stage and its adjoint, for the training path
 * of the pyramid.  Replace `downsampling_by_n` / `downsampling_by_2` (utils.py:73-124) and what
 * autograd derives from them.
 *   y  (B, Ly) = conv1d(x (B, L), fir (taps), stride=factor, padding=(taps-1)/2),
 *     Ly = (L + 2*((taps-1)/2) - taps) / factor + 1
 *   dx (B, L)  = the gradient of that w.r.t. x for an upstream gradient g (B, Ly)
 * All tensors fp32, contiguous rows with the given pitches. */
int nnab_fir_decimate(const float* x, int64_t B, int64_t L, int64_t x_pitch, const float* fir,
                      int taps, int factor, float* y, int64_t Ly, void* stream);
int nnab_fir_decimate_adjoint(const float* g, int64_t B, int64_t Ly, int64_t g_pitch,
                              const float* fir, int taps, int factor, float* dx, int64_t L,
                              void* stream);

size_t nnab_cqt_pyramid_workspace_bytes(int64_t B, int64_t L, int n_octaves, int early_factor,
                                        int max_width, int hop, int path);
/*   h_packed: HOST array of n_octaves DEVICE pointers to the nnab_pack_basis() copy of
 *     each bank (octave i's real/imag pair), or NULL / NULL entries = CUDA-core kernel
 *     for that octave.
 *   lowpass_packed / early_packed: nnab_pack_fir() copies or NULL.  With all packed
 *     inputs present the whole pyramid runs on the tensor cores: every anti-alias stage
 *     is a framed contraction whose epilogue writes the next level's padded bf16 planes. */
int nnab_cqt_pyramid_forward(const float* x, int64_t B, int64_t L, int64_t x_pitch,
                             int n_octaves, const float* const* h_k_real,
                             const float* const* h_k_imag, const void* const* h_packed,
                             const int32_t* h_widths,
                             int n_filters, const float* lowpass, const void* lowpass_packed,
                             const float* early_filter, const void* early_packed,
                             int early_factor, int hop, int pad_mode, int n_bins,
                             const float* scale, float scale_all, int out_format,
                             float sqrt_eps, float* out, int64_t T,
                             void* workspace, size_t ws_bytes, int path, void* stream);
/* 16-bit x: the all-tensor-core plans only (every packed input present, path != SIMT); the
 * per-octave plan decimates x on the CUDA cores and returns NNAB_EUNSUPPORTED. */
int nnab_cqt_pyramid_forward_ex(const void* x, int x_dtype, int64_t B, int64_t L, int64_t x_pitch,
                                int n_octaves, const float* const* h_k_real,
                                const float* const* h_k_imag, const void* const* h_packed,
                                const int32_t* h_widths,
                                int n_filters, const float* lowpass, const void* lowpass_packed,
                                const float* early_filter, const void* early_packed,
                                int early_factor, int hop, int pad_mode, int n_bins,
                                const float* scale, float scale_all, int out_format,
                                float sqrt_eps, float* out, int64_t T,
                                void* workspace, size_t ws_bytes, int path, void* stream);

/* ------------------------------------------------------------------------- *
 * STFT.inverse / iSTFT.forward — features/stft.py:15-63 (inverse_stft), :318-356,
 * :526-546; helpers utils.py:43-70 (SURVEY §8f "next" #2).
 *   X (B, f_in, T, 2) complex spectrogram; f_in = n_fft/2+1 with onesided, else n_fft
 *   kernel_cos / kernel_sin (n_fft, n_fft) = `kernel_cos_inv`/`kernel_sin_inv` of
 *     STFT(iSTFT=True) or `kernel_cos`/`kernel_sin` of the iSTFT module; packed once with
 *     nnab_pack_istft_basis (the one-sided mirroring of utils.py:63-70 is folded in)
 *   window (n_fft) = `window_mask`;  length < 0 means None
 *   out (B, out_len): out_len = n_fft + hop*(T-1) - 2*pad (length None, center) etc.
 * Runs on the tensor-core kernel only (inverse-DFT GEMM + overlap-add epilogue +
 * window-sumsquare normalisation).
 * ------------------------------------------------------------------------- */
size_t nnab_packed_istft_bytes(int n_fft, int f_in);
int nnab_pack_istft_basis(const float* kernel_cos, const float* kernel_sin, int n_fft, int f_in,
                          int onesided, void* packed, void* stream);
size_t nnab_istft_workspace_bytes(int64_t B, int f_in, int64_t T, int n_fft, int hop);
int nnab_istft_forward(const float* X, int64_t B, int f_in, int64_t T, const void* packed,
                       const float* window, int n_fft, int hop, int center, int64_t length,
                       float* out, int64_t out_len, void* workspace, size_t ws_bytes,
                       void* stream);

/* ------------------------------------------------------------------------- *
 * Input gradient of the framed complex contraction (SURVEY §8f "next" #1, the dX half;
 * the reference gets it from autograd through conv1d, stft.py:290-293 / cqt.py:749-750):
 *   g   (B, F, T, 2)  gradient w.r.t. (real, imag) = (conv(x, w_re), -conv(x, w_im))
 *   dx  (B, L)        = pad^T ( overlap_add_t ( g_re[., t] @ w_re - g_im[., t] @ w_im ) )
 * `packed_adj` = nnab_pack_adjoint_basis(w_re, w_im) (W^T rows, bf16 hi/lo).  One GEMM on
 * the tensor-core kernel with the overlap-add epilogue, then the padding adjoint.
 * ------------------------------------------------------------------------- */
size_t nnab_packed_adjoint_bytes(int K, int F);
int nnab_pack_adjoint_basis(const float* w_re, const float* w_im, int F, int K, void* packed,
                            void* stream);
size_t nnab_framed_backward_input_workspace_bytes(int64_t B, int64_t L, int K, int F, int hop,
                                                  int center);
int nnab_framed_backward_input(const float* g, int64_t B, int F, int64_t T, const void* packed_adj,
                               int K, int hop, int center, int pad_mode, float* dx, int64_t L,
                               void* workspace, size_t ws_bytes, void* stream);

/* Weight gradient of the framed complex contraction (the dW half of SURVEY §8f #1):
 *   dw (2F, K) fp32:  rows [0, F)  = sum_{b,t} g_re[b,f,t] * frame_{b,t}   (= d loss / d w_re)
 *                     rows [F, 2F) = sum_{b,t} g_im[b,f,t] * frame_{b,t}   (= -d loss / d w_im)
 * One split-K GEMM on the tensor-core kernel: gradient rows x transposed frame matrix. */
size_t nnab_framed_backward_weight_workspace_bytes(int64_t B, int64_t L, int K, int F, int hop,
                                                   int center);
int nnab_framed_backward_weight(const float* g, const float* x, int64_t B, int64_t L,
                                int64_t x_pitch, int F, int64_t T, int K, int hop, int center,
                                int pad_mode, float* dw, void* workspace, size_t ws_bytes,
                                void* stream);

/* The inverse STFT and both gradients above run one overlap-add GEMM of M_rows rows x F_out output samples
 * over K_gemm (rounded up to 64):
 *   nnab_framed_backward_input   M_rows = B*T, F_out = K,     K_gemm = 2F
 *   nnab_istft_forward           M_rows = B*T, F_out = n_fft, K_gemm = 2 f_in
 *   nnab_framed_backward_weight  M_rows = 2F,  F_out = K,     K_gemm = B*T rounded up to 64
 * K is cut into chunks of at most 4096 products per fp32 accumulator, at most k_splits_hint of them (64 for the
 * three calls): min(ceil(K_gemm / 4096), 64); the overlap-add atomics sum the chunks.  F_out is limited to 32768
 * (128 N tiles of 256 samples); above it the three calls return NNAB_EUNSUPPORTED before anything is enqueued.
 * Host only (tests): out[0..4] = supported (0 / 1), N tile width, N tiles, K chunks the launch uses, MMA flops it
 * executes (bf16 split terms and tile padding included). */
int nnab_debug_ola_plan(int F_out, int K_gemm, int64_t M_rows, int k_splits_hint, double* out);

/* ------------------------------------------------------------------------- *
 * Chunked streams: B streams that advance together, one push per chunk (DESIGN.md §3.10).
 * Each *_chunk_forward takes the arguments of the matching *_forward_ex with (x, L, x_pitch) replaced by
 *   state     DEVICE fp32 carry ring of nnab_chunk_state_bytes(B, K) bytes (K = n_fft or width), owned by
 *             the caller for the stream's lifetime (its contents need no initialisation)
 *   received, n_carry, frames   host counters: raw samples pushed before this chunk, how many of the last
 *             of them the ring carries, frames returned so far (0, 0, 0 for a new stream; the library
 *             returns NNAB_EINVAL for counters no stream can have)
 *   chunk, chunk_dtype, n, chunk_pitch   the new (B, n) samples (NNAB_DTYPE_*; chunk may be NULL iff n == 0)
 *   flush     1 on the last push: the remaining frames, with the right centre padding
 * T is the number of frames THIS push returns: every frame whose samples have all arrived (frame t needs
 * t*hop + K - pad of them, reflect padding also pad + 1), all remaining frames on flush.  The library
 * returns NNAB_EINVAL when T disagrees.  out holds those T frames in the offline layout.  The frames are
 * those the offline call gives for the whole stream, bit for bit on the tensor-core plans.  After the call
 * the caller advances its counters: received += n, frames += T,
 * n_carry = received - max(0, min(frames*hop - pad, pad > 0 ? received - pad - 1 : received)).
 * A push is the pool push (*_pool_forward below) of B lanes that share these counters, lane b in slot b: the
 * launches of the offline call on (B, (T - 1) * hop + K samples) when T > 0, then one carry launch (every row
 * returns T frames, so there is no mask launch).  The workspace queries equal *_pool_workspace_bytes(T > 0 ? B : 0,
 * T, ...) for the T this push returns.
 * Plans that read x as fp32 directly (SIMT) return NNAB_EUNSUPPORTED before anything is enqueued.
 * The MFCC call takes top_db < 0 (None) only: the floor is a maximum over the whole clip.
 * ------------------------------------------------------------------------- */
size_t nnab_chunk_state_bytes(int64_t B, int K);
size_t nnab_stft_chunk_workspace_bytes(int64_t B, int64_t received, int64_t frames, int64_t n, int flush,
                                       int n_fft, int F, int hop, int center, int pad_mode, int path);
int nnab_stft_chunk_forward(void* state, int64_t received, int64_t n_carry, int64_t frames, const void* chunk,
                            int chunk_dtype, int64_t B, int64_t n, int64_t chunk_pitch, int flush,
                            const float* wcos, const float* wsin, const void* packed, int n_fft, int F, int hop,
                            int center, int pad_mode, int out_format, float sqrt_eps, float* out, int64_t T,
                            void* workspace, size_t ws_bytes, int path, void* stream);
size_t nnab_filterbank_chunk_workspace_bytes(int64_t B, int64_t received, int64_t frames, int64_t n, int flush,
                                             int n_fft, int F, int hop, int center, int pad_mode, int n_fb,
                                             int path, int has_table);
int nnab_stft_filterbank_chunk_forward(void* state, int64_t received, int64_t n_carry, int64_t frames,
                                       const void* chunk, int chunk_dtype, int64_t B, int64_t n,
                                       int64_t chunk_pitch, int flush, const float* wcos, const float* wsin,
                                       const void* packed, int n_fft, int F, int hop, int center, int pad_mode,
                                       float sqrt_eps, float power, const float* fb, int n_fb,
                                       const void* fb_table, float* out, int64_t T, void* workspace,
                                       size_t ws_bytes, int path, void* stream);
size_t nnab_mfcc_chunk_workspace_bytes(int64_t B, int64_t received, int64_t frames, int64_t n, int flush,
                                       int n_fft, int F, int hop, int center, int pad_mode, int n_mels, int path,
                                       int has_table);
int nnab_mfcc_chunk_forward(void* state, int64_t received, int64_t n_carry, int64_t frames, const void* chunk,
                            int chunk_dtype, int64_t B, int64_t n, int64_t chunk_pitch, int flush,
                            const float* wcos, const float* wsin, const void* packed, int n_fft, int F, int hop,
                            int center, int pad_mode, float sqrt_eps, float power, const float* mel_basis,
                            int n_mels, const void* fb_table, float amin, float ref, float top_db,
                            const float* dct, int n_mfcc, float* out, int64_t T, void* workspace,
                            size_t ws_bytes, int path, void* stream);
size_t nnab_cqt1992v2_chunk_workspace_bytes(int64_t B, int64_t received, int64_t frames, int64_t n, int flush,
                                            int width, int n_bins, int hop, int center, int pad_mode, int path);
int nnab_cqt1992v2_chunk_forward(void* state, int64_t received, int64_t n_carry, int64_t frames,
                                 const void* chunk, int chunk_dtype, int64_t B, int64_t n, int64_t chunk_pitch,
                                 int flush, const float* k_real, const float* k_imag, const void* packed,
                                 const int32_t* h_k_begin, const int32_t* h_k_end, int n_bins, int width,
                                 int hop, int center, int pad_mode, const float* scale, float scale_all,
                                 int out_format, float sqrt_eps, float* out, int64_t T, void* workspace,
                                 size_t ws_bytes, int path, void* stream);

/* Stream pools: `slots` independent streams that advance by their own amounts (DESIGN.md §3.10).  Each
 * *_pool_forward takes the arguments of the matching *_chunk_forward with (received, n_carry, frames) and
 * flush replaced by a lane table, B by `slots` and T by T_max:
 *   state     DEVICE fp32 carry ring of nnab_chunk_state_bytes(slots, K) bytes; row s belongs to slot s
 *   lanes, d_lanes   the same n_lanes lanes, a HOST copy the library checks and a DEVICE copy the kernels
 *             read (the caller keeps both alive until the call's work has run).  One lane per slot that
 *             receives samples, ends, or returns frames in this push: its counters before the push (as for
 *             *_chunk_forward), n new samples chunk[slot, :n] and end = 1 on the stream's last push (its
 *             remaining frames, with the right padding, as flush).  The A lanes that return frames come
 *             first, then the others; slots ascend within each group and appear once.
 *   chunk, chunk_dtype, slots, n, chunk_pitch   the (slots, n) samples; every lane's n <= this n
 *   A, T_max  lanes that return frames and the most frames one of them returns
 * out is (A, ..., T_max) in the offline layout: row i holds lane i's new frames, bit for bit those of the
 * offline call on its whole stream (tensor-core plans), and exact zeros at t >= its count.  NNAB_EINVAL for
 * counters no stream can have, a slot out of range / repeated / out of order, a lane n above the chunk width,
 * an A or T_max that disagrees with the lanes, a lane with nothing to do, or an end on a stream too short for
 * its padding; all checks run before anything is enqueued.  The launches are those of the offline call on
 * (A, (T_max - 1) * hop + K samples), one carry launch and one mask launch; idle slots cost nothing.  After the
 * call the caller advances each lane's counters as for *_chunk_forward.  The SIMT plans return
 * NNAB_EUNSUPPORTED before anything is enqueued.  The workspace queries equal the offline queries for A clips
 * of (T_max - 1) * hop + K samples, uncentred (0 when A or T_max is 0). */
typedef struct nnab_stream_lane {
  int64_t slot, received, n_carry, frames, n, end;
} nnab_stream_lane;
size_t nnab_stft_pool_workspace_bytes(int64_t A, int64_t T_max, int n_fft, int F, int hop, int path);
int nnab_stft_pool_forward(void* state, const nnab_stream_lane* lanes, const nnab_stream_lane* d_lanes,
                           int64_t n_lanes, int64_t A, const void* chunk, int chunk_dtype, int64_t slots, int64_t n,
                           int64_t chunk_pitch, const float* wcos, const float* wsin, const void* packed, int n_fft,
                           int F, int hop, int center, int pad_mode, int out_format, float sqrt_eps, float* out,
                           int64_t T_max, void* workspace, size_t ws_bytes, int path, void* stream);
size_t nnab_filterbank_pool_workspace_bytes(int64_t A, int64_t T_max, int n_fft, int F, int hop, int n_fb,
                                            int path, int has_table);
int nnab_stft_filterbank_pool_forward(void* state, const nnab_stream_lane* lanes, const nnab_stream_lane* d_lanes,
                                      int64_t n_lanes, int64_t A, const void* chunk, int chunk_dtype, int64_t slots,
                                      int64_t n, int64_t chunk_pitch, const float* wcos, const float* wsin,
                                      const void* packed, int n_fft, int F, int hop, int center, int pad_mode,
                                      float sqrt_eps, float power, const float* fb, int n_fb, const void* fb_table,
                                      float* out, int64_t T_max, void* workspace, size_t ws_bytes, int path,
                                      void* stream);
size_t nnab_mfcc_pool_workspace_bytes(int64_t A, int64_t T_max, int n_fft, int F, int hop, int n_mels, int path,
                                      int has_table);
int nnab_mfcc_pool_forward(void* state, const nnab_stream_lane* lanes, const nnab_stream_lane* d_lanes,
                           int64_t n_lanes, int64_t A, const void* chunk, int chunk_dtype, int64_t slots, int64_t n,
                           int64_t chunk_pitch, const float* wcos, const float* wsin, const void* packed, int n_fft,
                           int F, int hop, int center, int pad_mode, float sqrt_eps, float power,
                           const float* mel_basis, int n_mels, const void* fb_table, float amin, float ref,
                           float top_db, const float* dct, int n_mfcc, float* out, int64_t T_max, void* workspace,
                           size_t ws_bytes, int path, void* stream);
size_t nnab_cqt1992v2_pool_workspace_bytes(int64_t A, int64_t T_max, int width, int n_bins, int hop, int path);
int nnab_cqt1992v2_pool_forward(void* state, const nnab_stream_lane* lanes, const nnab_stream_lane* d_lanes,
                                int64_t n_lanes, int64_t A, const void* chunk, int chunk_dtype, int64_t slots,
                                int64_t n, int64_t chunk_pitch, const float* k_real, const float* k_imag,
                                const void* packed, const int32_t* h_k_begin, const int32_t* h_k_end, int n_bins,
                                int width, int hop, int center, int pad_mode, const float* scale, float scale_all,
                                int out_format, float sqrt_eps, float* out, int64_t T_max, void* workspace,
                                size_t ws_bytes, int path, void* stream);

/* Streamed CQT pyramid: nnab_cqt_pyramid_forward_ex's arguments with (x, L, x_pitch) replaced by state, the
 * three host counters, the chunk and flush as above.
 *   state     DEVICE fp32, nnab_cqt_pyramid_chunk_state_bytes(B, n_octaves, widths, hop, early_factor) bytes:
 *             one ring per signal (the raw samples, then every decimated level); no initialisation needed
 *   n_carry   raw samples the raw ring carries: received - max(0, min(frames*hop - pad_0 [no early stage],
 *             received - pad_0 - 1 [no early stage], 128 d floor(R_1 / 128) - 128)), R_1 the final samples of
 *             the next signal and d its factor (DESIGN.md §3.10)
 * Before the end, sample n of a decimated signal is final once d n + c samples of its source have arrived
 * (d = 2, or early_factor for the early stage; c = 130 on the plan without early downsampling whose FIR-source
 * banks are 256 wide ("generation 2"), else 129), and T counts the frames final in every octave; on flush
 * every level gets its full length and T is the rest (octave frame counts that differ: NNAB_EINVAL).  The
 * pushes run the whole-clip call's tensor-core plan and kernels, so their frames equal it bit for bit.  A push is
 * the pool push (nnab_cqt_pyramid_pool_forward) of B lanes that share these counters, lane b in slot b: one plan
 * launch that writes the lanes' descriptors, then per signal its octave launches on the B rows (when T > 0), its
 * FIR stage launches and its carry launch, then one mask launch.  hop
 * must be a multiple of 2^(n_octaves - 1).  The SIMT path, a missing packed operand, or a launch outside the
 * kernels' limits returns NNAB_EUNSUPPORTED before anything is enqueued.  Both size queries are host-only. */
size_t nnab_cqt_pyramid_chunk_state_bytes(int64_t B, int n_octaves, const int32_t* widths, int hop,
                                          int early_factor);
size_t nnab_cqt_pyramid_chunk_workspace_bytes(int64_t B, int64_t received, int64_t n_carry, int64_t frames,
                                              int64_t n, int flush, int n_octaves, const int32_t* widths,
                                              int hop, int early_factor, int pad_mode);
int nnab_cqt_pyramid_chunk_forward(void* state, int64_t received, int64_t n_carry, int64_t frames,
                                   const void* chunk, int chunk_dtype, int64_t B, int64_t n, int64_t chunk_pitch,
                                   int flush, int n_octaves, const float* const* h_k_real,
                                   const float* const* h_k_imag, const void* const* h_packed,
                                   const int32_t* h_widths, int n_filters, const float* lowpass,
                                   const void* lowpass_packed, const float* early_filter, const void* early_packed,
                                   int early_factor, int hop, int pad_mode, int n_bins, const float* scale,
                                   float scale_all, int out_format, float sqrt_eps, float* out, int64_t T,
                                   void* workspace, size_t ws_bytes, int path, void* stream);
/* Host-only plan of one push (B = 1) for tests: per signal s (the raw samples first when early_factor > 1),
 * out[8 s ..] = final samples before and after the push, ring length, first sample kept after it, source origin
 * of its FIR stage and that stage's first output row (-1: the stage computes nothing), and the stage's CUDA-core
 * edge-fix windows of next-level outputs: head [R0 of s + 1, out[8 s + 6]) and tail [out[8 s + 7], R1 of s + 1)
 * (none: 0 / -1); then out[8 n_signals] = the frame bound after the push. */
int nnab_debug_pyramid_chunk_plan(int64_t received, int64_t n_carry, int64_t frames, int64_t n, int flush,
                                  int n_octaves, const int32_t* widths, int hop, int early_factor, int pad_mode,
                                  int64_t* out);

/* Pool of streamed CQT pyramids: the stream pools' (state, lanes, d_lanes, n_lanes, A, chunk, chunk_dtype, slots,
 * n, chunk_pitch) in front of nnab_cqt_pyramid_chunk_forward's pyramid arguments, then (out, T_max).  The state is
 * nnab_cqt_pyramid_chunk_state_bytes(slots, ...): row s of every signal's ring belongs to slot s.  A lane's n_carry
 * is the raw-ring carry of nnab_cqt_pyramid_chunk_forward and its `end` that call's flush; each lane is checked
 * by that call's rules (counters, frame bound, ring capacity, the octaves' frame counts at an end), the table by the
 * pools' (order, repeated slots, A, T_max, n above the chunk width), and every launch against the kernels' limits,
 * all before anything is enqueued.  Row i of out (A, n_bins, T_max[, 2]) holds lane i's frames, bit for bit those
 * of the whole-clip call on its stream, then exact zeros.  The launches are the chunk call's, the plan and mask
 * launches included, over the same stages on (n_lanes, ...) rows (the octaves on the A rows).  The workspace query
 * is host-only and takes the host lane table. */
size_t nnab_cqt_pyramid_pool_workspace_bytes(const nnab_stream_lane* lanes, int64_t n_lanes, int64_t A,
                                             int64_t T_max, int n_octaves, const int32_t* widths, int hop,
                                             int early_factor, int pad_mode);
int nnab_cqt_pyramid_pool_forward(void* state, const nnab_stream_lane* lanes, const nnab_stream_lane* d_lanes,
                                  int64_t n_lanes, int64_t A, const void* chunk, int chunk_dtype, int64_t slots,
                                  int64_t n, int64_t chunk_pitch, int n_octaves, const float* const* h_k_real,
                                  const float* const* h_k_imag, const void* const* h_packed,
                                  const int32_t* h_widths, int n_filters, const float* lowpass,
                                  const void* lowpass_packed, const float* early_filter, const void* early_packed,
                                  int early_factor, int hop, int pad_mode, int n_bins, const float* scale,
                                  float scale_all, int out_format, float sqrt_eps, float* out, int64_t T_max,
                                  void* workspace, size_t ws_bytes, int path, void* stream);
/* Host-only plan of one pool push for tests: for lane i, out[i (8 n_signals + 1) ..] in the layout of
 * nnab_debug_pyramid_chunk_plan, from the lane's (signal, lane) descriptors. */
int nnab_debug_pyramid_pool_plan(const nnab_stream_lane* lanes, int64_t n_lanes, int64_t A, int n_octaves,
                                 const int32_t* widths, int hop, int early_factor, int pad_mode, int64_t* out);

/* Streamed inverse STFT: nnab_istft_forward's arguments, with the frames of ONE push as X (B, f_in, T, 2)
 * (T may be 0) and in front of them
 *   state     DEVICE fp32, nnab_chunk_state_bytes(B, n_fft) bytes: the overlap-add partial sums later frames
 *             still reach (no initialisation needed)
 *   frames, emitted   host counters: frames pushed before X, output samples returned so far
 * and behind `center`: flush (1 on the last push) and length (< 0: None; read on flush only).
 * out receives the samples no later frame can change: overlap-add positions below (frames + T) * hop (and
 * below the earliest end the output can still have), the centre crop applied at the start; on flush the rest,
 * with the offline length / centre rules.  out_len must be that count; NNAB_EINVAL for counters no stream has
 * or a length shorter than the samples already returned.  Each sample is divided by the window sum-square of
 * its global position.  The concatenation equals nnab_istft_forward on all frames to fp32 rounding (both
 * overlap-add with fp32 atomics).  A push is the pool push (nnab_istft_pool_forward below) of B lanes that share
 * these counters, lane b in slot b with X row b: one seed launch, the FMT_OLA pre-pass and GEMM over B x T frames
 * (when T > 0) and one finalize launch.  The workspace query equals nnab_istft_pool_workspace_bytes(B, f_in, T,
 * n_fft, hop), so it includes the overlap-add rows' lead of n_fft positions. */
size_t nnab_istft_chunk_workspace_bytes(int64_t B, int f_in, int64_t T, int n_fft, int hop);
int nnab_istft_chunk_forward(void* state, int64_t frames, int64_t emitted, const float* X, int64_t B, int f_in,
                             int64_t T, const void* packed, const float* window, int n_fft, int hop, int center,
                             int flush, int64_t length, float* out, int64_t out_len, void* workspace,
                             size_t ws_bytes, void* stream);

/* Inverse STFT pools: `slots` independent streamed inverse STFTs that advance by their own frame counts
 * (DESIGN.md §3.10 "Inverse pools").  nnab_istft_chunk_forward's arguments with the counters, flush and length
 * moved into a lane table:
 *   state     DEVICE fp32, nnab_chunk_state_bytes(slots, n_fft) bytes; row s holds slot s's open partial sums
 *   lanes, d_lanes   the same n_lanes lanes, a HOST copy the library checks and a DEVICE copy the kernels read
 *             (the caller keeps both alive until the call's work has run).  One lane per slot that receives
 *             frames or ends in this push: its counters before the push (frames, emitted: as for
 *             *_chunk_forward), `row` = its row of X (-1: no new frames), T its new frames X[row, :, :T], end = 1
 *             on its last push and `length` (< 0: None; read only where end is set).  The A lanes that return
 *             samples come first, then the others; slots ascend within each group and appear once.
 *   X         (R, f_in, t, 2) fp32 frames, rows distinct between lanes; frames past a lane's T are never read
 *   A, n_max, T_max   lanes that return samples, the most samples one of them returns, the most frames one
 *             lane brings
 * out is (A, n_max): row i holds lane i's new samples, those nnab_istft_chunk_forward returns for the same
 * counters and frames, then exact zeros.  NNAB_EINVAL for counters no stream has (by the rules of
 * nnab_istft_chunk_forward, flush without any frame and a length shorter than the samples already returned
 * included), a slot out of range / repeated / out of order, a row out of range / repeated / not -1 exactly
 * when T = 0, T > t, an A, n_max or T_max that disagrees with the lanes, or a lane with nothing to do; all
 * checks run before anything is enqueued.  A push is one seed launch (the carried sums of every lane), the
 * FMT_OLA pre-pass and GEMM once over n_lanes x T_max frames, and one finalize launch (samples, zeros, carry);
 * idle slots cost nothing.  After the call the caller advances each lane's counters as for
 * *_chunk_forward.  The workspace query is 0 when n_lanes is 0, else
 * nnab_istft_workspace_bytes(n_lanes, f_in, max(T_max, 1), n_fft, hop) plus the overlap-add rows' lead of n_fft
 * positions: n_lanes rows of n_fft floats, each rounded up to 8 floats, the total to 256 bytes. */
typedef struct nnab_istft_lane {
  int64_t slot, row, frames, emitted, T, end, length;
} nnab_istft_lane;
size_t nnab_istft_pool_workspace_bytes(int64_t n_lanes, int f_in, int64_t T_max, int n_fft, int hop);
int nnab_istft_pool_forward(void* state, const nnab_istft_lane* lanes, const nnab_istft_lane* d_lanes,
                            int64_t n_lanes, int64_t A, int64_t slots, const float* X, int64_t R, int f_in, int64_t t,
                            const void* packed, const float* window, int n_fft, int hop, int center, float* out,
                            int64_t n_max, int64_t T_max, void* workspace, size_t ws_bytes, void* stream);

/* Device-planned pools (DESIGN.md §3.10 "Device pools"): the stream pools and the inverse STFT pool with every
 * per-push number on the DEVICE, so that a push reads nothing on the host, has one fixed geometry and can be
 * captured in a CUDA graph.  All slots are computed on every push: row s of every output is slot s.
 *   counters  DEVICE int64 (3, slots): forward pools received, frames, ended; the inverse pool frames, emitted,
 *             ended.  Zero for fresh streams; the push advances them, nnab_pool_device_reset zeroes masked slots.
 *   errors, error_info   DEVICE int32 (slots) and int64 (slots, 2): a slot whose push the host pool would refuse is
 *             dropped whole (counters, ring / state untouched, zero frames) and errors[s] records the first such
 *             NNAB_LANE_* code, error_info[s] its values, until the slot's reset.  The other slots proceed.
 *   counts    DEVICE int32 (slots): frames (samples) row s holds after the push; the rest of the row is zeros.
 *   d_lanes   DEVICE scratch of `slots` lanes that the plan launch writes and the pool kernels read.
 * One plan launch (one thread per slot, the host checks' own functions) writes the lanes, counts, codes and the
 * advanced counters; an idle, ended or dropped slot gets an all-zero lane, which returns nothing and carries
 * nothing.  Then the body of the matching *_pool_forward runs with n_lanes = A = slots. */
enum {
  NNAB_LANE_OK = 0,
  NNAB_LANE_ELENGTH = 1,   /* lengths[s] (counts[s]) outside [0, chunk width (frames of X)]; info: the value */
  NNAB_LANE_EENDED = 2,    /* samples / frames or an end for an ended stream                               */
  NNAB_LANE_ESHORT = 3,    /* an end on a stream too short for the module; info: its length                 */
  NNAB_LANE_ENOFRAMES = 4, /* inverse: an end on a stream without frames                                     */
  NNAB_LANE_ELENGTH_SHORT = 5 /* inverse: length shorter than the samples returned; info: length, emitted   */
};
/* T_cap: the most frames one push of at most `chunk` samples can return (an end included), for framing (K, hop,
 * pad, pad_mode).  n_cap: the most samples one inverse push of at most `frames` frames can return (a flush with
 * any length included).  Host only; 0 for arguments no pool takes. */
int64_t nnab_pool_frame_cap(int64_t chunk, int K, int hop, int pad, int pad_mode);
int64_t nnab_istft_pool_sample_cap(int64_t frames, int n_fft, int hop, int center);
/* Forward: the *_pool_forward arguments with (lanes, d_lanes, n_lanes, A) replaced by (counters, lengths, end,
 * errors, error_info, counts, d_lanes): lengths DEVICE int32 (slots), end DEVICE uint8 (slots).  n is the fixed
 * chunk width, T_max must be nnab_pool_frame_cap(n, ...) and out is (slots, ..., T_max).  The workspace is
 * *_pool_workspace_bytes(slots, T_max, ...).  Only host-side arguments are checked (NNAB_EINVAL).  The SIMT plans
 * return NNAB_EUNSUPPORTED with only the plan launch enqueued: a push with every length 0 and no end then changes
 * nothing, which is how a caller can probe the route. */
int nnab_stft_pool_device_forward(void* state, int64_t* counters, const int32_t* lengths, const uint8_t* end,
                                  int32_t* errors, int64_t* error_info, int32_t* counts, nnab_stream_lane* d_lanes,
                                  const void* chunk, int chunk_dtype, int64_t slots, int64_t n, int64_t chunk_pitch,
                                  const float* wcos, const float* wsin, const void* packed, int n_fft, int F, int hop,
                                  int center, int pad_mode, int out_format, float sqrt_eps, float* out, int64_t T_max,
                                  void* workspace, size_t ws_bytes, int path, void* stream);
int nnab_stft_filterbank_pool_device_forward(void* state, int64_t* counters, const int32_t* lengths,
                                             const uint8_t* end, int32_t* errors, int64_t* error_info,
                                             int32_t* counts, nnab_stream_lane* d_lanes, const void* chunk,
                                             int chunk_dtype, int64_t slots, int64_t n, int64_t chunk_pitch,
                                             const float* wcos, const float* wsin, const void* packed, int n_fft,
                                             int F, int hop, int center, int pad_mode, float sqrt_eps, float power,
                                             const float* fb, int n_fb, const void* fb_table, float* out,
                                             int64_t T_max, void* workspace, size_t ws_bytes, int path, void* stream);
int nnab_mfcc_pool_device_forward(void* state, int64_t* counters, const int32_t* lengths, const uint8_t* end,
                                  int32_t* errors, int64_t* error_info, int32_t* counts, nnab_stream_lane* d_lanes,
                                  const void* chunk, int chunk_dtype, int64_t slots, int64_t n, int64_t chunk_pitch,
                                  const float* wcos, const float* wsin, const void* packed, int n_fft, int F, int hop,
                                  int center, int pad_mode, float sqrt_eps, float power, const float* mel_basis,
                                  int n_mels, const void* fb_table, float amin, float ref, float top_db,
                                  const float* dct, int n_mfcc, float* out, int64_t T_max, void* workspace,
                                  size_t ws_bytes, int path, void* stream);
int nnab_cqt1992v2_pool_device_forward(void* state, int64_t* counters, const int32_t* lengths, const uint8_t* end,
                                       int32_t* errors, int64_t* error_info, int32_t* counts,
                                       nnab_stream_lane* d_lanes, const void* chunk, int chunk_dtype, int64_t slots,
                                       int64_t n, int64_t chunk_pitch, const float* k_real, const float* k_imag,
                                       const void* packed, const int32_t* h_k_begin, const int32_t* h_k_end,
                                       int n_bins, int width, int hop, int center, int pad_mode, const float* scale,
                                       float scale_all, int out_format, float sqrt_eps, float* out, int64_t T_max,
                                       void* workspace, size_t ws_bytes, int path, void* stream);
/* Inverse: X (slots, f_in, t, 2) fp32, row s slot s's frames; frame_counts DEVICE int32 (slots) its new frames
 * X[s, :, :frame_counts[s]]; end DEVICE uint8 and length DEVICE int64 (slots; < 0: None).  out is (slots, n_max)
 * with n_max = nnab_istft_pool_sample_cap(t, ...); the workspace nnab_istft_pool_workspace_bytes(slots, f_in, t,
 * n_fft, hop). */
int nnab_istft_pool_device_forward(void* state, int64_t* counters, const int32_t* frame_counts, const uint8_t* end,
                                   const int64_t* length, int32_t* errors, int64_t* error_info, int32_t* counts,
                                   nnab_istft_lane* d_lanes, int64_t slots, const float* X, int f_in, int64_t t,
                                   const void* packed, const float* window, int n_fft, int hop, int center,
                                   float* out, int64_t n_max, void* workspace, size_t ws_bytes, void* stream);
/* New streams in the slots where mask[s] != 0 (mask NULL: every slot): their counters, errors and error_info
 * become zero.  One launch; the ring / state needs no clearing (a fresh lane reads none of it). */
int nnab_pool_device_reset(int64_t* counters, int32_t* errors, int64_t* error_info, const uint8_t* mask,
                           int64_t slots, void* stream);
/* Host-only runs of the plan launches for tests, on HOST arrays of the layouts above (counters advanced in
 * place; lanes written as int64 rows of 6 / 7). */
int nnab_debug_device_pool_plan(int64_t* counters, const int32_t* lengths, const uint8_t* end, int32_t* errors,
                                int64_t* error_info, int32_t* counts, nnab_stream_lane* lanes, int64_t slots,
                                int64_t n, int K, int hop, int pad, int pad_mode);
int nnab_debug_device_istft_plan(int64_t* counters, const int32_t* frame_counts, const uint8_t* end,
                                 const int64_t* length, int32_t* errors, int64_t* error_info, int32_t* counts,
                                 nnab_istft_lane* lanes, int64_t slots, int64_t t, int n_fft, int hop, int center);

/* Device-planned pool of streamed CQT pyramids (DESIGN.md §3.10 "Device pyramid pools"): nnab_cqt_pyramid_pool_forward
 * with (lanes, d_lanes, n_lanes, A) replaced by the device pools' (counters, lengths, end, errors, error_info, counts,
 * d_lanes); counters are received, frames, ended per slot, a lane's n_carry is derived from them.  n is the fixed
 * chunk width; T_max must be caps[0] of nnab_cqt_pyramid_pool_device_caps(n, ...) and out is (slots, n_bins,
 * T_max[, 2]).  A slot whose push PyramidPool would refuse is dropped (NNAB_LANE_ELENGTH, NNAB_LANE_EENDED, or
 * NNAB_LANE_ESHORT for an end the stream is too short for; info: its length).  Every stage and octave launches on
 * every push over all slots at the caps, so the launch list does not depend on the traffic.  Only host-side
 * arguments are checked; the SIMT path, a missing packed operand or a launch outside the kernels' limits returns
 * NNAB_EUNSUPPORTED before anything is enqueued.
 * The caps query (host only) fills caps[0] = T_cap, the most frames one push of at most `chunk` samples returns
 * (an end included), caps[1 + s] = the most FIR outputs stage s -> s + 1 computes for one lane from its first
 * 128-output row (0 for the last signal), caps[1 + n_signals + s] = the most samples one push stores into signal
 * s's ring; n_signals = n_octaves (+ 1 with early_factor > 1).  It is NNAB_EINVAL if a push without an end could be
 * refused, which the ring bounds exclude.  The workspace query is host-only (0 for arguments no pool takes). */
int nnab_cqt_pyramid_pool_device_caps(int64_t chunk, int n_octaves, const int32_t* widths, int hop,
                                      int early_factor, int pad_mode, int64_t* caps);
size_t nnab_cqt_pyramid_pool_device_workspace_bytes(int64_t slots, int64_t chunk, int n_octaves,
                                                    const int32_t* widths, int hop, int early_factor, int pad_mode);
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
                                         int path, void* stream);
/* Host-only run of its plan launch for tests (nnab_debug_device_pool_plan's layout). */
int nnab_debug_device_pyramid_plan(int64_t* counters, const int32_t* lengths, const uint8_t* end, int32_t* errors,
                                   int64_t* error_info, int32_t* counts, nnab_stream_lane* lanes, int64_t slots,
                                   int64_t n, int n_octaves, const int32_t* widths, int hop, int early_factor,
                                   int pad_mode);

/* Per-channel energy normalisation (PCEN; beyond the reference, DESIGN.md §3.11).  E is a non-negative (B, C, T)
 * fp32 spectrogram; per row (b, c), with the parameters of channel c:
 *   M[t] = (1 - s) M[t-1] + s E[t]          M[-1] = E[0]
 *   P[t] = bias^power expm1(power log1p(E[t] (eps + M[t])^-gain / bias))
 * The parameters s, gain, bias, power are DEVICE fp32 arrays: param_stride 1 reads element c (C of them),
 * param_stride 0 element 0 (scalars).  Their values are not checked (0 < s <= 1, gain >= 0, bias > 0, power > 0
 * are the caller's); eps must be > 0.  Each row is a sequential fp32 recurrence in frame order, so a row split
 * into several streamed calls gives the same bits as one call.
 *
 * nnab_pcen_forward writes P (B, C, T).  Training: M (non-NULL) receives the (B, C, T) smoother output for
 * nnab_pcen_backward; state must then be NULL.  Streaming: state (slots, C) fp32 and primed (slots, C) uint8
 * carry each slot's last M; row b belongs to slot row_slot[b] (DEVICE int32, NULL: slot b, then B <= slots) and
 * advances by counts[b] frames (DEVICE int32, clamped to [0, T]; NULL: T), its P zero past them.  A slot that is
 * not primed starts from its first frame as the offline call does; a row with frames leaves its slot primed.
 * Rows must map to distinct slots; a row mapped outside [0, slots) computes nothing.  counts and row_slot need
 * state.  One launch; T == 0 or B == 0 enqueues nothing. */
int nnab_pcen_forward(const float* E, int64_t B, int C, int64_t T, const float* s, const float* gain,
                      const float* bias, const float* power, int param_stride, float eps, float* P, float* M,
                      float* state, uint8_t* primed, int64_t slots, const int32_t* row_slot, const int32_t* counts,
                      void* stream);
/* Workspace of nnab_pcen_backward with grad_params: the per-row parameter partials (4 B C floats). */
size_t nnab_pcen_workspace_bytes(int64_t B, int C);
/* Adjoint of the offline call: grad_P (B, C, T) -> grad_E (B, C, T) (NULL: not written) and grad_params (4, n)
 * with n = C (param_stride 1) or 1, rows in the order s, gain, bias, power (NULL: not computed; otherwise the
 * workspace is required).  M is the training forward's output.  The parameter sums run in a fixed order (no
 * atomics): two calls give the same bits.  One launch, plus one for grad_params. */
int nnab_pcen_backward(const float* E, const float* M, const float* grad_P, int64_t B, int C, int64_t T,
                       const float* s, const float* gain, const float* bias, const float* power, int param_stride,
                       float eps, float* grad_E, float* grad_params, void* workspace, size_t ws_bytes, void* stream);
/* Un-prime the stream slots where mask[s] != 0 (mask NULL: every slot) of a (slots, C) primed array.  One
 * launch; reads nothing on the host, so it can be captured in a CUDA graph. */
int nnab_pcen_reset(uint8_t* primed, const uint8_t* mask, int64_t slots, int C, void* stream);

/* Kernel launches issued by this library since load (process wide; used by
 * bench.py for its `gpu_launches` claim). */
uint64_t nnab_launch_count(void);

/* Leave `n_sms` SMs out of the persistent tensor-core grids (process wide, default 0) so
 * that a concurrently running collective (the NCCL output gather of the multi-GPU path)
 * has SMs to run on; returns the previous value.  Any n_sms >= 0 is kept (a negative value
 * becomes 0); a persistent grid never drops below one CTA, so a reserve of at least the
 * device's SM count runs every persistent kernel on a single CTA. */
int nnab_set_sm_reserve(int n_sms);

/* Persistent-grid ledger: the persistent tensor-core launches enqueued since the last read (process
 * wide), their summed CTAs, and the smallest and largest grid among them.  Writes each non-NULL
 * pointer, then resets the ledger; with no launch since the last read all four are 0.  Counted on
 * the host at launch, so replaying a captured CUDA graph counts nothing.  Returns NNAB_OK. */
int nnab_persistent_grid_read(uint64_t* launches, uint64_t* ctas, int* min_grid, int* max_grid);

/* Live timing of the dominant kernel (the framed contraction) for bench.py's
 * roofline: while enabled, every framed-contraction launch is bracketed by a
 * cudaEvent pair recorded on the launching stream.  nnab_profile_read()
 * synchronises those events, returns the summed duration in ms and the number
 * of launches timed since the last read, and resets the accumulator. */
void nnab_profile_enable(int on);
int nnab_profile_read(double* framed_ms, uint64_t* framed_launches);
/* MMA flops the tensor-core launches EXECUTED since the last read (all bf16 split terms, tile
 * padding and structural zeros included) -> bench.py's roofline.tensor_pipe. */
int nnab_profile_read_exec_flops(double* exec_flops);
/* Launches of the tall-A CQT kernel that ran the balanced schedule (tiles shared between two
 * CTAs, framed_tct_kernel<., true>) since load -- lets a test tell which schedule it exercised. */
uint64_t nnab_balanced_launch_count(void);
/* Launches of the block-partial STFT kernel that ran with separate MMA and epilogue warps
 * (framed_tcb_ws_kernel: four phases, fused filterbank or operand planes, nb <= 88) since load.  The
 * plain four-phase kernel executes the same MMA flops at the same width; this tells the two apart. */
uint64_t nnab_block_ws_launch_count(void);

/* Routes of nnab_cqt_pyramid_forward(_ex), counted since load so that a test can tell which one a call took.
 * Each counter grows by one per successful enqueue of its stage, inside that entry point only: the plan once
 * per call, an octave route once per octave, a FIR route once per decimation stage (the early stage included).
 * The chunk, pool and device-pool entry points run the same kernels and count in nnab_stream_route_count. */
enum {
  NNAB_PYR_PLAN_GEN2 = 0,         /* one plane set per level, banded FIR stages                         */
  NNAB_PYR_PLAN_GEN1 = 1,         /* early downsampling and any bank width, dense FIR stages             */
  NNAB_PYR_PLAN_PER_OCTAVE = 2,   /* octave by octave on fp32 levels, CUDA-core FIR stages               */
  NNAB_PYR_OCT_KERNEL = 3,        /* the octave kernel (resident bank, frame phases) on the level planes */
  NNAB_PYR_OCT_DENSE_PLANES = 4,  /* the dense tensor-core kernel on the level planes (hop % 8 == 0)     */
  NNAB_PYR_OCT_DENSE_FP32 = 5,    /* the dense tensor-core kernel on the fp32 level, split per frame phase */
  NNAB_PYR_OCT_TC_LOOP = 6,       /* per-octave plan: the dense tensor-core kernel                       */
  NNAB_PYR_OCT_SIMT = 7,          /* per-octave plan: the SIMT kernel                                    */
  NNAB_PYR_FIR_BANDED = 8,        /* gen-2: banded tensor-core FIR stage with its clip-edge fix          */
  NNAB_PYR_FIR_DENSE = 9,         /* gen-1: FIR stage on the dense tensor-core kernel                    */
  NNAB_PYR_FIR_SIMT = 10,         /* per-octave plan: CUDA-core FIR stage                                */
  NNAB_PYR_ROUTES = 11
};
/* The counter of `route` (an NNAB_PYR_* value); 0 for any other value. */
uint64_t nnab_pyramid_route_count(int route);

/* Kernel routes of nnab_cqt1992v2_forward(_ex), counted since load so that a test can tell which one a call took.
 * Each successful call adds one to the counter of the route it enqueued (a dense call once, however many frame
 * phases it launches).  The chunk, pool and device-pool entry points count in nnab_stream_route_count. */
enum {
  NNAB_CQ1992_TALL = 0,           /* tall-A kernel (8-bin-group bank), static schedule                  */
  NNAB_CQ1992_TALL_BALANCED = 1,  /* tall-A kernel, balanced schedule (nnab_balanced_launch_count)      */
  NNAB_CQ1992_VARN = 2,           /* per-K-block-width kernel (8-bin-group bank the tall kernel refuses) */
  NNAB_CQ1992_VARN_SPLITK = 3,    /* the same, K cut into chunks, then the split-K finalize             */
  NNAB_CQ1992_DENSE = 4,          /* dense tensor-core kernel, one launch per frame phase               */
  NNAB_CQ1992_DENSE_SPLITK = 5,   /* the same with K cut into chunks, then the split-K finalize         */
  NNAB_CQ1992_SIMT = 6,           /* CUDA-core kernel                                                   */
  NNAB_CQ1992_ROUTES = 7
};
/* The counter of `route` (an NNAB_CQ1992_* value); 0 for any other value. */
uint64_t nnab_cqt1992v2_route_count(int route);

/* Routes of nnab_stft_forward(_ex), nnab_stft_filterbank_forward(_ex) and nnab_mfcc_forward(_ex), counted since
 * load so that a test can tell which one a call took.  Each successful call adds one to the counter of the
 * contraction route it enqueued (a dense call once, however many frame phases it launches); a filterbank or MFCC
 * call also adds one to the counter of its filterbank route.  The chunk, pool and device-pool entry points count
 * in nnab_stream_route_count. */
enum {
  NNAB_STFT_BLOCK = 0,         /* block-partial kernel (periodic-Hann DFT basis)                         */
  NNAB_STFT_DENSE = 1,         /* dense tensor-core kernel, one launch per frame phase                   */
  NNAB_STFT_DENSE_SPLITK = 2,  /* the same with K cut into chunks, then the split-K finalize             */
  NNAB_STFT_SIMT = 3,          /* CUDA-core kernel                                                       */
  NNAB_STFT_FB_FUSED = 4,      /* filterbank summed in the contraction's epilogue (banded table)         */
  NNAB_STFT_FB_PLANES = 5,     /* |X| ** power as bf16 operand planes, then a tensor-core GEMM with the bank */
  NNAB_STFT_FB_GEMM = 6,       /* fp32 (B, F, T) power spectrogram, then the CUDA-core filterbank GEMM   */
  NNAB_STFT_ROUTES = 7
};
/* The counter of `route` (an NNAB_STFT_* value); 0 for any other value. */
uint64_t nnab_stft_route_count(int route);

/* Routes of the streamed calls, counted apart from the offline counters above so that a test can tell which kernels
 * a push took.  The chunk, pool and device-pool entry points of STFT, filterbank, MFCC and CQT1992v2 count as their
 * offline calls do (family NNAB_ROUTES_STFT or NNAB_ROUTES_CQ1992, the same route values); the three pyramid stream
 * calls count the plan once per push, an octave route per octave and a FIR route per decimation stage they launch
 * (family NNAB_ROUTES_PYR).  A push counts after it succeeds, and only when it returns frames: a push of no frames, or
 * one refused with NNAB_EUNSUPPORTED, counts nothing, and no push moves an offline counter.  A device-pool push counts
 * when it is enqueued; replaying a captured CUDA graph of it counts nothing. */
enum { NNAB_ROUTES_STFT = 0, NNAB_ROUTES_CQ1992 = 1, NNAB_ROUTES_PYR = 2 };
/* The stream counter of `route` in `family` (an NNAB_ROUTES_* value); 0 for any other pair. */
uint64_t nnab_stream_route_count(int family, int route);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif

#ifdef __cplusplus
}
#endif
#endif /* NNAB_H_ */
