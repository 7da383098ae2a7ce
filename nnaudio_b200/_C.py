"""ctypes binding of ``libnnab.so`` (C ABI in ``include/nnab.h``).

PyTorch is used only for device memory and the current CUDA stream; every
compute call goes through the C ABI with raw device pointers.  There is no
CPU / eager fallback: if the library is missing, or a tensor is not a CUDA
fp32 tensor (a waveform may also be bfloat16 or float16), the call fails loudly.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int32, c_int64, c_size_t, c_uint64, c_void_p

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libnnab.so")

PAD_REFLECT, PAD_CONSTANT = 0, 1
FMT_MAGNITUDE, FMT_COMPLEX, FMT_PHASE_ANGLE, FMT_PHASE_UNIT = 0, 1, 2, 3
PATH_AUTO, PATH_SIMT, PATH_TCGEN05 = 0, 1, 2
DTYPE_F32, DTYPE_BF16, DTYPE_F16 = 0, 1, 2
EUNSUPPORTED = -6

# sample types of the waveform the forward entry points read (NNAB_DTYPE_*)
_WAVE_DTYPES = {torch.float32: DTYPE_F32, torch.bfloat16: DTYPE_BF16, torch.float16: DTYPE_F16}

# "tc" = the wgmma/TMA tensor-core kernels; "tcgen05" (the C constant's name) means the same
_PATH_NAMES = {"auto": PATH_AUTO, "simt": PATH_SIMT, "tc": PATH_TCGEN05, "tcgen05": PATH_TCGEN05}

# every symbol include/nnab.h declares: (restype, argtypes)
_P = c_void_p
SIGNATURES = {
    "nnab_abi_version": (c_int, []),
    "nnab_strerror": (c_char_p, [c_int]),
    "nnab_last_cuda_error": (c_char_p, []),
    "nnab_launch_count": (c_uint64, []),
    "nnab_set_sm_reserve": (c_int, [c_int]),
    "nnab_persistent_grid_read": (c_int, [_P, _P, _P, _P]),
    "nnab_profile_enable": (None, [c_int]),
    "nnab_profile_read": (c_int, [_P, _P]),
    "nnab_profile_read_exec_flops": (c_int, [_P]),
    "nnab_balanced_launch_count": (c_uint64, []),
    "nnab_block_ws_launch_count": (c_uint64, []),
    "nnab_pyramid_route_count": (c_uint64, [c_int]),
    "nnab_cqt1992v2_route_count": (c_uint64, [c_int]),
    "nnab_stft_route_count": (c_uint64, [c_int]),
    "nnab_stream_route_count": (c_uint64, [c_int, c_int]),
    "nnab_pack_tile_n": (c_int, [c_int]),
    "nnab_packed_basis_bytes": (c_size_t, [c_int, c_int]),
    "nnab_pack_basis": (c_int, [_P, _P, c_int, c_int, _P, _P]),
    "nnab_stft_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int, c_int, c_int, c_int, c_int]),
    "nnab_stft_forward": (
        c_int,
        [_P, c_int64, c_int64, c_int64, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int,
         c_float, _P, c_int64, _P, c_size_t, c_int, _P],
    ),
    "nnab_filterbank_table_bytes": (c_size_t, [c_int]),
    "nnab_build_filterbank_table": (c_int, [_P, c_int, c_int, _P, _P, _P]),
    "nnab_filterbank_table_fuses": (c_int, [_P, _P, c_int]),
    "nnab_filterbank_workspace_bytes": (
        c_size_t, [c_int64, c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    "nnab_stft_filterbank_forward": (
        c_int,
        [_P, c_int64, c_int64, c_int64, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float,
         c_float, _P, c_int, _P, _P, c_int64, _P, c_size_t, c_int, _P],
    ),
    "nnab_mfcc_workspace_bytes": (
        c_size_t, [c_int64, c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    "nnab_mfcc_forward": (
        c_int,
        [_P, c_int64, c_int64, c_int64, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float,
         c_float, _P, c_int, _P, c_float, c_float, c_float, _P, c_int, _P, c_int64, _P, c_size_t,
         c_int, _P],
    ),
    "nnab_cqt1992v2_workspace_bytes": (
        c_size_t, [c_int64, c_int64, c_int, c_int, c_int, c_int, c_int]),
    "nnab_cqt1992v2_forward": (
        c_int,
        [_P, c_int64, c_int64, c_int64, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int,
         _P, c_float, c_int, c_float, _P, c_int64, _P, c_size_t, c_int, _P],
    ),
    "nnab_packed_istft_bytes": (c_size_t, [c_int, c_int]),
    "nnab_pack_istft_basis": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P]),
    "nnab_istft_workspace_bytes": (c_size_t, [c_int64, c_int, c_int64, c_int, c_int]),
    "nnab_istft_forward": (
        c_int,
        [_P, c_int64, c_int, c_int64, _P, _P, c_int, c_int, c_int, c_int64, _P, c_int64, _P,
         c_size_t, _P],
    ),
    "nnab_packed_adjoint_bytes": (c_size_t, [c_int, c_int]),
    "nnab_pack_adjoint_basis": (c_int, [_P, _P, c_int, c_int, _P, _P]),
    "nnab_framed_backward_input_workspace_bytes": (
        c_size_t, [c_int64, c_int64, c_int, c_int, c_int, c_int]),
    "nnab_framed_backward_input": (
        c_int,
        [_P, c_int64, c_int, c_int64, _P, c_int, c_int, c_int, c_int, _P, c_int64, _P, c_size_t, _P],
    ),
    "nnab_framed_backward_weight_workspace_bytes": (
        c_size_t, [c_int64, c_int64, c_int, c_int, c_int, c_int]),
    "nnab_framed_backward_weight": (
        c_int,
        [_P, _P, c_int64, c_int64, c_int64, c_int, c_int64, c_int, c_int, c_int, c_int, _P, _P,
         c_size_t, _P],
    ),
    "nnab_pack_basis_ex": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P]),
    "nnab_block_layout_ok": (c_int, [c_int, c_int]),
    "nnab_stream_write_value32": (c_int, [_P, _P, ctypes.c_uint32]),
    "nnab_stream_wait_value32_geq": (c_int, [_P, _P, ctypes.c_uint32]),
    "nnab_packed_block_bytes": (c_size_t, [c_int, c_int]),
    "nnab_pack_basis_block": (c_int, [c_int, c_int, _P, _P]),
    "nnab_debug_varn_plan": (c_int, [_P, _P, c_int, c_int, c_int, _P, _P, _P, _P, _P]),
    "nnab_debug_ola_plan": (c_int, [c_int, c_int, c_int64, c_int, _P]),
    "nnab_fir_decimate": (c_int, [_P, c_int64, c_int64, c_int64, _P, c_int, c_int, _P, c_int64, _P]),
    "nnab_fir_decimate_adjoint": (
        c_int, [_P, c_int64, c_int64, c_int64, _P, c_int, c_int, _P, c_int64, _P]),
    "nnab_packed_fir_bytes": (c_size_t, [c_int, c_int]),
    "nnab_pack_fir": (c_int, [_P, c_int, c_int, _P, _P]),
    "nnab_cqt_pyramid_workspace_bytes": (
        c_size_t, [c_int64, c_int64, c_int, c_int, c_int, c_int, c_int]),
    "nnab_cqt_pyramid_forward": (
        c_int,
        [_P, c_int64, c_int64, c_int64, c_int, _P, _P, _P, _P, c_int, _P, _P, _P, _P, c_int, c_int,
         c_int, c_int, _P, c_float, c_int, c_float, _P, c_int64, _P, c_size_t, c_int, _P],
    ),
}
# the *_ex forward entry points: the same arguments, (x, x_dtype) in place of x
for _name in ("nnab_stft_forward", "nnab_stft_filterbank_forward", "nnab_mfcc_forward",
              "nnab_cqt1992v2_forward", "nnab_cqt_pyramid_forward"):
    _res, _args = SIGNATURES[_name]
    SIGNATURES[_name + "_ex"] = (_res, [_P, c_int] + _args[1:])
# the *_chunk_forward entry points: (state, received, n_carry, frames, chunk, chunk_dtype, B, n, chunk_pitch,
# flush) in place of (x, B, L, x_pitch); their workspace queries take (B, received, frames, n, flush) in place
# of (B, L) and the pad mode after `center`
_CHUNK_HEAD = [_P, c_int64, c_int64, c_int64, _P, c_int, c_int64, c_int64, c_int64, c_int]
_CHUNK_WS_HEAD = [c_int64, c_int64, c_int64, c_int64, c_int]
_POOL_HEAD = [_P, _P, _P, c_int64, c_int64, _P, c_int, c_int64, c_int64, c_int64]
_DEVICE_HEAD = [_P] * 9 + [c_int, c_int64, c_int64, c_int64]
SIGNATURES["nnab_chunk_state_bytes"] = (c_size_t, [c_int64, c_int])
for _name, _ws in (("nnab_stft_forward", "nnab_stft"), ("nnab_stft_filterbank_forward", "nnab_filterbank"),
                   ("nnab_mfcc_forward", "nnab_mfcc"), ("nnab_cqt1992v2_forward", "nnab_cqt1992v2")):
    _res, _args = SIGNATURES[_name]
    SIGNATURES[_name.replace("_forward", "_chunk_forward")] = (_res, _CHUNK_HEAD + _args[4:])
    _wres, _wargs = SIGNATURES[_ws + "_workspace_bytes"]
    SIGNATURES[_ws + "_chunk_workspace_bytes"] = (_wres, _CHUNK_WS_HEAD + _wargs[2:6] + [c_int] + _wargs[6:])
    # the *_pool_forward entry points: (state, lanes, d_lanes, n_lanes, A, chunk, chunk_dtype, slots, n,
    # chunk_pitch) in place of (x, B, L, x_pitch); their workspace queries take (A, T_max) in place of (B, L)
    # and no `center`
    SIGNATURES[_name.replace("_forward", "_pool_forward")] = (_res, _POOL_HEAD + _args[4:])
    SIGNATURES[_ws + "_pool_workspace_bytes"] = (_wres, [c_int64, c_int64] + _wargs[2:5] + _wargs[6:])
    # the *_pool_device_forward entry points: (state, counters, lengths, end, errors, error_info, counts,
    # d_lanes, chunk, chunk_dtype, slots, n, chunk_pitch) in place of (x, B, L, x_pitch)
    SIGNATURES[_name.replace("_forward", "_pool_device_forward")] = (_res, _DEVICE_HEAD + _args[4:])
SIGNATURES["nnab_pool_frame_cap"] = (c_int64, [c_int64, c_int, c_int, c_int, c_int])
SIGNATURES["nnab_istft_pool_sample_cap"] = (c_int64, [c_int64, c_int, c_int, c_int])
SIGNATURES["nnab_istft_pool_device_forward"] = (
    c_int, [_P] * 9 + [c_int64, _P, c_int, c_int64, _P, _P, c_int, c_int, c_int, _P, c_int64, _P, c_size_t, _P])
SIGNATURES["nnab_pool_device_reset"] = (c_int, [_P, _P, _P, _P, c_int64, _P])
SIGNATURES["nnab_debug_device_pool_plan"] = (c_int, [_P] * 7 + [c_int64, c_int64, c_int, c_int, c_int, c_int])
SIGNATURES["nnab_debug_device_istft_plan"] = (c_int, [_P] * 8 + [c_int64, c_int64, c_int, c_int, c_int])
SIGNATURES["nnab_cqt_pyramid_chunk_state_bytes"] = (c_size_t, [c_int64, c_int, _P, c_int, c_int])
SIGNATURES["nnab_cqt_pyramid_chunk_workspace_bytes"] = (
    c_size_t, [c_int64, c_int64, c_int64, c_int64, c_int64, c_int, c_int, _P, c_int, c_int, c_int])
SIGNATURES["nnab_cqt_pyramid_chunk_forward"] = (
    c_int, _CHUNK_HEAD + SIGNATURES["nnab_cqt_pyramid_forward"][1][4:])
SIGNATURES["nnab_debug_pyramid_chunk_plan"] = (
    c_int, [c_int64, c_int64, c_int64, c_int64, c_int, c_int, _P, c_int, c_int, c_int, _P])
# pyramid pools: the pool head in front of the chunk call's pyramid arguments; the workspace query and the debug
# plan take the host lane table
SIGNATURES["nnab_cqt_pyramid_pool_forward"] = (c_int, _POOL_HEAD + SIGNATURES["nnab_cqt_pyramid_forward"][1][4:])
SIGNATURES["nnab_cqt_pyramid_pool_workspace_bytes"] = (
    c_size_t, [_P, c_int64, c_int64, c_int64, c_int, _P, c_int, c_int, c_int])
SIGNATURES["nnab_debug_pyramid_pool_plan"] = (c_int, [_P, c_int64, c_int64, c_int, _P, c_int, c_int, c_int, _P])
# device pyramid pools: the device head in front of the pyramid arguments; the caps, workspace and debug plan queries
# take the geometry (chunk, n_octaves, widths, hop, early_factor, pad_mode)
_PYR_GEOMETRY = [c_int, _P, c_int, c_int, c_int]
SIGNATURES["nnab_cqt_pyramid_pool_device_forward"] = (
    c_int, _DEVICE_HEAD + SIGNATURES["nnab_cqt_pyramid_forward"][1][4:])
SIGNATURES["nnab_cqt_pyramid_pool_device_caps"] = (c_int, [c_int64] + _PYR_GEOMETRY + [_P])
SIGNATURES["nnab_cqt_pyramid_pool_device_workspace_bytes"] = (c_size_t, [c_int64, c_int64] + _PYR_GEOMETRY)
SIGNATURES["nnab_debug_device_pyramid_plan"] = (c_int, [_P] * 7 + [c_int64, c_int64] + _PYR_GEOMETRY)
SIGNATURES["nnab_istft_chunk_workspace_bytes"] = SIGNATURES["nnab_istft_workspace_bytes"]
SIGNATURES["nnab_istft_chunk_forward"] = (
    c_int, [_P, c_int64, c_int64, _P, c_int64, c_int, c_int64, _P, _P, c_int, c_int, c_int, c_int, c_int64, _P,
            c_int64, _P, c_size_t, _P])
SIGNATURES["nnab_istft_pool_workspace_bytes"] = SIGNATURES["nnab_istft_workspace_bytes"]
SIGNATURES["nnab_istft_pool_forward"] = (
    c_int, [_P, _P, _P, c_int64, c_int64, c_int64, _P, c_int64, c_int, c_int64, _P, _P, c_int, c_int, c_int, _P,
            c_int64, c_int64, _P, c_size_t, _P])

_lib = None


def lib() -> ctypes.CDLL:
    """Load ``libnnab.so`` once; raise (never fall back) when it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found: the CUDA extension must be built first "
                "(python -c 'import __graft_entry__ as g; g.build()' or "
                "nnaudio_b200/csrc/build.sh). nnaudio_b200 has no CPU fallback."
            )
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if a declared symbol is missing
            fn.restype = res
            fn.argtypes = args
        if handle.nnab_abi_version() != 1:
            raise ImportError("libnnab.so ABI version mismatch")
        _lib = handle
    return _lib


def default_path() -> int:
    """Kernel family selector; ``NNAUDIO_B200_PATH=auto|simt|tc``."""
    return _PATH_NAMES[os.environ.get("NNAUDIO_B200_PATH", "auto").lower()]


def resolve_path(path) -> int:
    if path is None:
        return default_path()
    if isinstance(path, str):
        return _PATH_NAMES[path.lower()]
    return int(path)


def launch_count() -> int:
    return int(lib().nnab_launch_count())


def balanced_launch_count() -> int:
    """Tall-A CQT launches that ran the balanced (shared-tile) schedule since load."""
    return int(lib().nnab_balanced_launch_count())


def block_ws_launch_count() -> int:
    """Block-partial STFT launches that ran the warp-specialised kernel (separate MMA and epilogue warps) since
    load."""
    return int(lib().nnab_block_ws_launch_count())


# routes of nnab_cqt_pyramid_forward (NNAB_PYR_*): the plan, each octave's kernel, each FIR stage's kernel
(PYR_PLAN_GEN2, PYR_PLAN_GEN1, PYR_PLAN_PER_OCTAVE, PYR_OCT_KERNEL, PYR_OCT_DENSE_PLANES, PYR_OCT_DENSE_FP32,
 PYR_OCT_TC_LOOP, PYR_OCT_SIMT, PYR_FIR_BANDED, PYR_FIR_DENSE, PYR_FIR_SIMT) = range(11)
PYR_ROUTES = 11


def pyramid_route_count(route: int) -> int:
    """Stages of the offline CQT pyramid call that took ``route`` (a PYR_* constant) since load; the streaming
    and pool calls count in stream_route_count."""
    return int(lib().nnab_pyramid_route_count(int(route)))


# kernel routes of nnab_cqt1992v2_forward (NNAB_CQ1992_*)
(CQ1992_TALL, CQ1992_TALL_BALANCED, CQ1992_VARN, CQ1992_VARN_SPLITK, CQ1992_DENSE, CQ1992_DENSE_SPLITK,
 CQ1992_SIMT) = range(7)
CQ1992_ROUTES = 7


def cqt1992v2_route_count(route: int) -> int:
    """Offline CQT1992v2 calls that took kernel route ``route`` (a CQ1992_* constant) since load; the streaming
    and pool calls count in stream_route_count."""
    return int(lib().nnab_cqt1992v2_route_count(int(route)))


# routes of nnab_stft_forward / nnab_stft_filterbank_forward / nnab_mfcc_forward (NNAB_STFT_*): the contraction's
# kernel, then (filterbank and MFCC calls) how the bank was applied
(STFT_BLOCK, STFT_DENSE, STFT_DENSE_SPLITK, STFT_SIMT, STFT_FB_FUSED, STFT_FB_PLANES, STFT_FB_GEMM) = range(7)
STFT_ROUTES = 7


def stft_route_count(route: int) -> int:
    """Offline STFT / filterbank / MFCC calls that took route ``route`` (a STFT_* constant) since load; the
    streaming and pool calls count in stream_route_count."""
    return int(lib().nnab_stft_route_count(int(route)))


# counter families of nnab_stream_route_count: each takes its offline counterpart's route values
ROUTES_STFT, ROUTES_CQ1992, ROUTES_PYR = 0, 1, 2


def stream_route_count(family: int, route: int) -> int:
    """Pushes of the chunk, pool and device-pool calls that took ``route`` since load, in ``family`` (ROUTES_STFT
    with a STFT_* route, ROUTES_CQ1992 with a CQ1992_* route, ROUTES_PYR with a PYR_* route).  Only a successful push
    that returns frames counts; a replayed CUDA graph counts nothing."""
    return int(lib().nnab_stream_route_count(int(family), int(route)))


def set_sm_reserve(n_sms: int) -> int:
    """Keep ``n_sms`` SMs out of the persistent kernels' grids (for a concurrent collective); returns the previous
    reserve.  The grids never drop below one CTA."""
    return int(lib().nnab_set_sm_reserve(int(n_sms)))


def persistent_grid_read():
    """(launches, summed CTAs, min grid, max grid) of the persistent tensor-core launches enqueued since the last
    read, then resets them; all zero when nothing launched.  Counted at launch: a replayed CUDA graph counts
    nothing."""
    n, c = c_uint64(0), c_uint64(0)
    lo, hi = c_int(0), c_int(0)
    _check(lib().nnab_persistent_grid_read(ctypes.byref(n), ctypes.byref(c), ctypes.byref(lo), ctypes.byref(hi)),
           "nnab_persistent_grid_read")
    return int(n.value), int(c.value), int(lo.value), int(hi.value)


def profile_enable(on: bool):
    lib().nnab_profile_enable(1 if on else 0)


def profile_read():
    """(summed ms, launches) of the framed-contraction kernel since the last read."""
    ms = ctypes.c_double(0.0)
    n = c_uint64(0)
    _check(lib().nnab_profile_read(ctypes.byref(ms), ctypes.byref(n)), "nnab_profile_read")
    return ms.value, int(n.value)


def profile_read_exec_flops() -> float:
    v = ctypes.c_double(0.0)
    _check(lib().nnab_profile_read_exec_flops(ctypes.byref(v)), "nnab_profile_read_exec_flops")
    return float(v.value)


def _check(rc: int, what: str):
    if rc != 0:
        L = lib()
        msg = L.nnab_strerror(rc).decode()
        if rc == -4:
            msg += ": " + L.nnab_last_cuda_error().decode()
        raise RuntimeError(f"{what} failed: {msg} (status {rc})")


def _dev_f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor")
    if not t.is_cuda:
        raise RuntimeError(
            f"{name} is on {t.device}: nnaudio_b200 runs only on CUDA (sm_90a) tensors; "
            "there is no CPU fallback"
        )
    if t.dtype != torch.float32:
        raise RuntimeError(f"{name} must be float32, got {t.dtype}")
    return t


def _dev_wave(t: torch.Tensor, name: str) -> torch.Tensor:
    """``_dev_f32`` for a waveform: float32, bfloat16 or float16."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor")
    if not t.is_cuda:
        raise RuntimeError(
            f"{name} is on {t.device}: nnaudio_b200 runs only on CUDA (sm_90a) tensors; "
            "there is no CPU fallback"
        )
    if t.dtype not in _WAVE_DTYPES:
        raise RuntimeError(f"{name} must be float32, bfloat16 or float16, got {t.dtype}")
    return t


def _ptr(t):
    return c_void_p(t.data_ptr()) if t is not None else None


def _stream(device) -> c_void_p:
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _workspace(nbytes: int, device):
    if nbytes <= 0:
        return None, 0
    ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
    return ws, nbytes


MAX_BATCH = 65535  # clips per C call (the pre-pass kernels put the clip index in gridDim.y)


# --------------------------------------------------------------------------- #
# caller-provided output buffers (multi-GPU gather: the kernels write straight into the slice of a
# symmetric-memory buffer; see nnaudio_b200.parallel)
# --------------------------------------------------------------------------- #
import threading as _threading

_OUT = _threading.local()


class output_into:
    """``with _C.output_into(buf): y = module(x)`` -- the forward call that runs inside writes its
    result into ``buf`` (a contiguous fp32 CUDA tensor of exactly the result's shape) instead of
    allocating one, and returns ``buf``.  Used once: the first matching allocation takes it."""

    def __init__(self, buf: torch.Tensor):
        self.buf = buf

    def __enter__(self):
        _OUT.buf = self.buf
        return self

    def __exit__(self, *exc):
        _OUT.buf = None
        return False


def _new_out(shape, device) -> torch.Tensor:
    buf = getattr(_OUT, "buf", None)
    if buf is not None and tuple(buf.shape) == tuple(shape) and buf.device == device \
            and buf.dtype == torch.float32 and buf.is_contiguous():
        _OUT.buf = None
        return buf
    return torch.empty(shape, dtype=torch.float32, device=device)


def _batch_chunked(fn):
    """Forward wrappers take any batch size: more than ``MAX_BATCH`` clips are run as several C
    calls on the same stream and concatenated (every op of the path is per-clip, including the
    MFCC ``top_db`` clamp)."""
    import functools

    @functools.wraps(fn)
    def wrapper(x, *args, **kwargs):
        if x.dim() != 2 or x.shape[0] <= MAX_BATCH:
            return fn(x, *args, **kwargs)
        return torch.cat([fn(x[i:i + MAX_BATCH], *args, **kwargs)
                          for i in range(0, x.shape[0], MAX_BATCH)], 0)

    return wrapper


def _batch_starts(B: int):
    """First clip of each C call of a ``B``-clip batch (the training and inverse wrappers split like
    ``_batch_chunked``)."""
    return range(0, B, MAX_BATCH)


def _as_rows(x: torch.Tensor):
    if x.dim() != 2:
        raise ValueError("internal: expected (B, L)")
    if x.stride(-1) != 1 or (x.shape[0] > 1 and x.stride(0) < x.shape[1]):
        x = x.contiguous()
    pitch = x.stride(0) if x.shape[0] > 1 else x.shape[1]
    return x, x.shape[0], x.shape[1], pitch


def _rows(x: torch.Tensor):
    """(B, L) fp32 view with unit inner stride -> (tensor, B, L, pitch)."""
    return _as_rows(_dev_f32(x, "x"))


def _wave_rows(x: torch.Tensor):
    """``_rows`` of a waveform in any sample type the forward entry points take
    -> (tensor, B, L, pitch, NNAB dtype).  A 16-bit waveform is passed on as is (no fp32 copy)."""
    x, B, L, pitch = _as_rows(_dev_wave(x, "x"))
    return x, B, L, pitch, _WAVE_DTYPES[x.dtype]


def _call_wave(call, x, pitch, dtype, strict_dtype):
    """``call(x, pitch, dtype)`` -> status of a forward entry point.  When the plan the library chose
    cannot read a 16-bit waveform (NNAB_EUNSUPPORTED, returned before anything is enqueued: the SIMT
    kernels, the per-octave CQT pyramid), run it once more on the float32 upcast; ``strict_dtype``
    (tests) turns that into an error instead, so a 16-bit route that is missing cannot hide."""
    rc = call(x, pitch, dtype)
    if rc == EUNSUPPORTED and dtype != DTYPE_F32 and not strict_dtype:
        x, _, _, pitch = _as_rows(x.float())
        rc = call(x, pitch, DTYPE_F32)
    return rc


# --------------------------------------------------------------------------- #
# basis packing (tensor-core path)
# --------------------------------------------------------------------------- #
LAYOUT_DENSE, LAYOUT_GROUPS = 0, 3


def pack_basis(w_re: torch.Tensor, w_im: torch.Tensor, layout: int = LAYOUT_DENSE):
    """bf16 hi/lo split of an (F, K) fp32 basis pair in the TMA/wgmma layout, or
    ``None`` when the library has no tensor-core kernel for it.  ``layout``: LAYOUT_GROUPS for long
    nested CQT banks (per-K-block-width / tall-A kernels)."""
    L = lib()
    F, K = w_re.shape
    nbytes = L.nnab_packed_basis_bytes(F, K)
    if nbytes == 0:
        return None
    packed = torch.empty(nbytes, dtype=torch.uint8, device=w_re.device)
    with torch.cuda.device(w_re.device):
        if layout == LAYOUT_DENSE:
            rc = L.nnab_pack_basis(_ptr(w_re), _ptr(w_im), F, K, _ptr(packed), _stream(w_re.device))
        else:
            rc = L.nnab_pack_basis_ex(_ptr(w_re), _ptr(w_im), F, K, int(layout), _ptr(packed),
                                      _stream(w_re.device))
        _check(rc, "nnab_pack_basis")
    return packed


def stream_write_value32(stream: torch.cuda.Stream, addr: int, value: int):
    """Stream-ordered 32-bit store to a (possibly peer-mapped) device address: a front-end memory
    operation, no kernel and no SM (cuStreamWriteValue32)."""
    _check(lib().nnab_stream_write_value32(ctypes.c_void_p(stream.cuda_stream), ctypes.c_void_p(addr),
                                           int(value) & 0xFFFFFFFF), "nnab_stream_write_value32")


def stream_wait_value32_geq(stream: torch.cuda.Stream, addr: int, value: int):
    """Work queued on ``stream`` after this waits until (int32)(*addr - value) >= 0 (cuStreamWaitValue32)."""
    _check(lib().nnab_stream_wait_value32_geq(ctypes.c_void_p(stream.cuda_stream), ctypes.c_void_p(addr),
                                              int(value) & 0xFFFFFFFF), "nnab_stream_wait_value32_geq")


def block_layout_ok(n_fft: int, hop: int) -> bool:
    return bool(lib().nnab_block_layout_ok(int(n_fft), int(hop)))


def pack_basis_block(w_re: torch.Tensor, hop: int):
    """Packed rows of the block-partial STFT kernel for an (F, n_fft) periodic-Hann DFT basis
    (the caller has checked the buffers with ``is_hann_dft``); generated analytically on the device."""
    L = lib()
    F, K = w_re.shape
    packed = torch.empty(L.nnab_packed_block_bytes(int(K), int(hop)), dtype=torch.uint8, device=w_re.device)
    with torch.cuda.device(w_re.device):
        _check(L.nnab_pack_basis_block(int(K), int(hop), _ptr(packed), _stream(w_re.device)),
               "nnab_pack_basis_block")
    return packed


def pack_fir(fir: torch.Tensor, dec: int):
    """Banded-Toeplitz bf16 hi/lo packing of a decimation FIR (tensor-core pyramid)."""
    L = lib()
    taps = fir.numel()
    packed = torch.empty(L.nnab_packed_fir_bytes(taps, dec), dtype=torch.uint8, device=fir.device)
    with torch.cuda.device(fir.device):
        _check(L.nnab_pack_fir(_ptr(fir), taps, dec, _ptr(packed), _stream(fir.device)),
               "nnab_pack_fir")
    return packed


def build_filterbank_table(fb: torch.Tensor):
    """Banded (<= 2 non-zeros per FFT bin) table of an (n_fb, F) filterbank for the
    fused tensor-core epilogue, or ``None`` when the bank is denser (e.g. gammatone).
    Init-time: synchronises the current stream once."""
    L = lib()
    n_fb, F = fb.shape
    table = torch.empty(L.nnab_filterbank_table_bytes(F), dtype=torch.uint8, device=fb.device)
    max_nnz = ctypes.c_int(0)
    with torch.cuda.device(fb.device):
        _check(L.nnab_build_filterbank_table(_ptr(fb), n_fb, F, _ptr(table), ctypes.byref(max_nnz),
                                             _stream(fb.device)), "nnab_build_filterbank_table")
    return table if max_nnz.value <= 2 else None


# --------------------------------------------------------------------------- #
# the framed transforms (STFT, filterbank, MFCC, CQT1992v2): one argument spec each, read by every call mode.
# A forward call is (waveform head, transform tail, out, T, workspace, workspace bytes, path, stream); the heads
# differ by mode (SIGNATURES), the tail is the same in all four.  The workspace queries take (K, F, hop) after
# their own head, then `center` (offline, chunk), the pad mode (chunk) and the transform's query tail.
# --------------------------------------------------------------------------- #
def _kb(k):
    return k.ctypes.data_as(c_void_p) if k is not None else None


class _Spec:
    """The C names and argument rules of one framed transform; ``kw`` holds its offline call's arguments."""

    def __init__(self, stem, ws, shape, geometry, tail, ws_tail):
        self.shape = shape        # (rows, T, kw) -> output shape
        self.geometry = geometry  # kw -> (K, F, hop) of the workspace queries
        self.tail = tail          # kw -> the arguments between the waveform head and `out`
        self.ws_tail = ws_tail    # (kw, path) -> the workspace query's arguments after its geometry
        self.forward, self.ws = f"nnab_{stem}_forward_ex", f"nnab_{ws}_workspace_bytes"
        self.chunk, self.chunk_ws = f"nnab_{stem}_chunk_forward", f"nnab_{ws}_chunk_workspace_bytes"
        self.pool, self.pool_ws = f"nnab_{stem}_pool_forward", f"nnab_{ws}_pool_workspace_bytes"
        self.device = f"nnab_{stem}_pool_device_forward"


def _stft_geometry(kw):
    return kw["n_fft"], kw["wcos"].shape[0], kw["hop"]


def _stft_head(kw):
    return (_ptr(kw["wcos"]), _ptr(kw["wsin"]), _ptr(kw["packed"]), kw["n_fft"], kw["wcos"].shape[0], kw["hop"],
            int(kw["center"]), kw["pad_mode"])


def _has_table(kw):
    """The workspace queries' ``has_table``: the call sums the bank in the contraction's epilogue."""
    t = kw.get("fb_table")
    return int(t is not None and lib().nnab_filterbank_table_fuses(_ptr(t), _ptr(kw["packed"]), kw["n_fft"]) != 0)


def _complex_shape(rows, bins, T, complex_out):
    return (rows, bins, T, 2) if complex_out else (rows, bins, T)


_SPECS = {
    "stft_forward": _Spec(
        "stft", "stft",
        lambda B, T, kw: _complex_shape(B, kw["wcos"].shape[0], T, kw["out_format"] == FMT_COMPLEX),
        _stft_geometry,
        lambda kw: _stft_head(kw) + (kw["out_format"], kw["sqrt_eps"]),
        lambda kw, path: (path,)),
    "stft_filterbank_forward": _Spec(
        "stft_filterbank", "filterbank",
        lambda B, T, kw: (B, kw["fb"].shape[0], T),
        _stft_geometry,
        lambda kw: _stft_head(kw) + (kw["sqrt_eps"], kw["power"], _ptr(kw["fb"]), kw["fb"].shape[0],
                                     _ptr(kw.get("fb_table"))),
        lambda kw, path: (kw["fb"].shape[0], path, _has_table(kw))),
    "mfcc_forward": _Spec(
        "mfcc", "mfcc",
        lambda B, T, kw: (B, kw["dct"].shape[0], T),
        _stft_geometry,
        lambda kw: _stft_head(kw) + (kw["sqrt_eps"], kw["power"], _ptr(kw["mel_basis"]), kw["mel_basis"].shape[0],
                                     _ptr(kw.get("fb_table")), kw["amin"], kw["ref"],
                                     -1.0 if kw["top_db"] is None else float(kw["top_db"]), _ptr(kw["dct"]),
                                     kw["dct"].shape[0]),
        lambda kw, path: (kw["mel_basis"].shape[0], path, _has_table(kw))),
    "cqt1992v2_forward": _Spec(
        "cqt1992v2", "cqt1992v2",
        lambda B, T, kw: _complex_shape(B, kw["k_real"].shape[0], T, kw["out_format"] != FMT_MAGNITUDE),
        lambda kw: (kw["k_real"].shape[1], kw["k_real"].shape[0], kw["hop"]),
        lambda kw: (_ptr(kw["k_real"]), _ptr(kw["k_imag"]), _ptr(kw["packed"]), _kb(kw["k_begin"]),
                    _kb(kw["k_end"]), kw["k_real"].shape[0], kw["k_real"].shape[1], kw["hop"], int(kw["center"]),
                    kw["pad_mode"], _ptr(kw["scale"]), kw["scale_all"], kw["out_format"], kw["sqrt_eps"]),
        lambda kw, path: (path,)),
}


def _offline(name, x, kw):
    spec, L = _SPECS[name], lib()
    x, B, Ln, pitch, dt = _wave_rows(x)
    K, F, hop = spec.geometry(kw)
    pad = K // 2 if kw["center"] else 0
    T = (Ln + 2 * pad - K) // hop + 1
    out = _new_out(spec.shape(B, T, kw), x.device)
    path = resolve_path(kw["path"])
    tail = spec.tail(kw)
    fn = getattr(L, spec.forward)
    with torch.cuda.device(x.device):
        ws, wsb = _workspace(getattr(L, spec.ws)(B, Ln, K, F, hop, int(kw["center"]), *spec.ws_tail(kw, path)),
                             x.device)
        rc = _call_wave(lambda xs, p, d: fn(_ptr(xs), d, B, Ln, p, *tail, _ptr(out), T, _ptr(ws), wsb, path,
                                            _stream(x.device)), x, pitch, dt, kw["strict_dtype"])
    _check(rc, spec.forward)
    return out


# x of the forward calls: a float32, bfloat16 or float16 (B, L) CUDA tensor; the output is float32.
@_batch_chunked
def stft_forward(x, wcos, wsin, packed, n_fft, hop, center, pad_mode, out_format, sqrt_eps,
                 path=None, strict_dtype=False):
    return _offline("stft_forward", x, locals())


@_batch_chunked
def stft_filterbank_forward(x, wcos, wsin, packed, n_fft, hop, center, pad_mode, sqrt_eps, power,
                            fb, fb_table=None, path=None, strict_dtype=False):
    return _offline("stft_filterbank_forward", x, locals())


@_batch_chunked
def mfcc_forward(x, wcos, wsin, packed, n_fft, hop, center, pad_mode, sqrt_eps, power, mel_basis,
                 amin, ref, top_db, dct, fb_table=None, path=None, strict_dtype=False):
    return _offline("mfcc_forward", x, locals())


@_batch_chunked
def cqt1992v2_forward(x, k_real, k_imag, packed, k_begin, k_end, hop, center, pad_mode, scale,
                      scale_all, out_format, sqrt_eps, path=None, strict_dtype=False):
    """k_begin / k_end: host int32 numpy arrays (per-bin support) or None."""
    return _offline("cqt1992v2_forward", x, locals())


def _bank_arrays(banks_real, banks_imag, packed):
    """The pyramid's per-octave C arrays: bank pointers (real, imaginary), packed bases (NULL where absent) and
    bank widths."""
    n = len(banks_real)
    return ((c_void_p * n)(*[t.data_ptr() for t in banks_real]),
            (c_void_p * n)(*[t.data_ptr() for t in banks_imag]),
            (c_void_p * n)(*[(t.data_ptr() if t is not None else None) for t in packed]),
            (c_int32 * n)(*[int(t.shape[1]) for t in banks_real]))


@_batch_chunked
def cqt_pyramid_forward(x, banks_real, banks_imag, packed, lowpass, lowpass_packed, early_filter,
                        early_packed, early_factor, hop, pad_mode, n_bins, scale, scale_all,
                        out_format, sqrt_eps, T, path=None, strict_dtype=False):
    """banks_*: lists (octave 0 = top) of (n_filters, width_i) fp32 CUDA tensors;
    packed: list of packed-basis tensors (or None entries) per octave."""
    L = lib()
    x, B, Ln, pitch, dt = _wave_rows(x)
    n_oct = len(banks_real)
    n_filters = banks_real[0].shape[0]
    re_arr, im_arr, pk_arr, widths = _bank_arrays(banks_real, banks_imag, packed)
    max_width = max(widths)
    out = _new_out(_complex_shape(B, n_bins, T, out_format != FMT_MAGNITUDE), x.device)
    path = resolve_path(path)
    with torch.cuda.device(x.device):
        ws, wsb = _workspace(
            L.nnab_cqt_pyramid_workspace_bytes(B, Ln, n_oct, early_factor, max_width, hop, path),
            x.device)
        rc = _call_wave(lambda xs, p, d: L.nnab_cqt_pyramid_forward_ex(
            _ptr(xs), d, B, Ln, p, n_oct, re_arr, im_arr, pk_arr, widths, n_filters,
            _ptr(lowpass), _ptr(lowpass_packed), _ptr(early_filter), _ptr(early_packed),
            early_factor, hop, pad_mode, n_bins, _ptr(scale),
            scale_all, out_format, sqrt_eps, _ptr(out), T, _ptr(ws), wsb, path, _stream(x.device)),
            x, pitch, dt, strict_dtype)
    _check(rc, "nnab_cqt_pyramid_forward_ex")
    return out


# --------------------------------------------------------------------------- #
# chunk calls (nnaudio_b200.streaming): one push of B streams.  `st` carries the device carry ring
# (st.ring, nnab_chunk_state_bytes) and the host counters (st.received, st.n_carry, st.frames); `x` is the
# (B, n) chunk or None; T the frames this push returns.  The remaining arguments are those of the offline
# call above.  Returns the frames, or None when the plan cannot read a chunk (NNAB_EUNSUPPORTED, nothing
# enqueued): the caller then takes the concat route.
# --------------------------------------------------------------------------- #
def chunk_state_bytes(B: int, K: int) -> int:
    return int(lib().nnab_chunk_state_bytes(int(B), int(K)))


def _chunk_args(st, x):
    """(chunk, n, pitch, NNAB sample type) of a push: the chunk's type, or the stream's when there is no chunk
    (a flush)."""
    if x is None:
        return None, 0, 0, _WAVE_DTYPES[st.dtype]
    if x.shape[-1] == 0:
        return None, 0, 0, _WAVE_DTYPES[x.dtype]
    x, _, n, pitch, dt = _wave_rows(x)
    return x, n, pitch, dt


def _chunk_result(rc, out, what):
    if rc == EUNSUPPORTED:
        return None
    _check(rc, what)
    return out


def _chunk(name, st, x, flush, T, kw):
    spec, L = _SPECS[name], lib()
    xs, n, pitch, dt = _chunk_args(st, x)
    B, dev = st.batch, st.ring.device
    out = torch.empty(spec.shape(B, T, kw), dtype=torch.float32, device=dev)
    path = resolve_path(kw["path"])
    with torch.cuda.device(dev):
        ws, wsb = _workspace(getattr(L, spec.chunk_ws)(B, st.received, st.frames, n, int(flush), *spec.geometry(kw),
                                                       int(kw["center"]), kw["pad_mode"], *spec.ws_tail(kw, path)), dev)
        rc = getattr(L, spec.chunk)(
            _ptr(st.ring), st.received, st.n_carry, st.frames, _ptr(xs), dt, B, n, pitch, int(flush), *spec.tail(kw),
            _ptr(out), T, _ptr(ws), wsb, path, _stream(dev))
    return _chunk_result(rc, out, spec.chunk)


def stft_chunk_forward(st, x, flush, T, wcos, wsin, packed, n_fft, hop, center, pad_mode, out_format, sqrt_eps,
                       path=None):
    return _chunk("stft_forward", st, x, flush, T, locals())


def stft_filterbank_chunk_forward(st, x, flush, T, wcos, wsin, packed, n_fft, hop, center, pad_mode, sqrt_eps,
                                  power, fb, fb_table=None, path=None):
    return _chunk("stft_filterbank_forward", st, x, flush, T, locals())


def mfcc_chunk_forward(st, x, flush, T, wcos, wsin, packed, n_fft, hop, center, pad_mode, sqrt_eps, power,
                       mel_basis, amin, ref, top_db, dct, fb_table=None, path=None):
    return _chunk("mfcc_forward", st, x, flush, T, locals())


def cqt1992v2_chunk_forward(st, x, flush, T, k_real, k_imag, packed, k_begin, k_end, hop, center, pad_mode, scale,
                            scale_all, out_format, sqrt_eps, path=None):
    return _chunk("cqt1992v2_forward", st, x, flush, T, locals())


# --------------------------------------------------------------------------- #
# pool calls (nnaudio_b200.streaming.StreamPool): one push of a stream pool.  `pool` carries the device carry
# ring (pool.ring, one row per slot) and pool.slots; `lanes` is the push's (n_lanes, 6) int64 lane table
# (nnab_stream_lane rows, the A lanes with frames first); `x` the (slots, n) chunk.  The remaining arguments are
# those of the offline call.  Returns the (A, ..., T_max) frames, or None when the plan cannot read a chunk
# (NNAB_EUNSUPPORTED, nothing enqueued).
# --------------------------------------------------------------------------- #
LANE_FIELDS = ("slot", "received", "n_carry", "frames", "n", "end")


def _lane_copies(lanes, device):
    """Host and device copies of a lane table: the host copy in pinned memory, the device copy made from it
    without blocking (torch's host allocator keeps the pinned block until the copy has run)."""
    if len(lanes) == 0:
        return None, None
    host = torch.as_tensor(lanes, dtype=torch.int64).contiguous().pin_memory()
    return host, host.to(device, non_blocking=True)


def _pool(name, pool, lanes, x, A, T_max, kw):
    spec, L = _SPECS[name], lib()
    xs, n, pitch, dt = _chunk_args(pool, x)
    dev = pool.ring.device
    out = torch.empty(spec.shape(A, T_max, kw), dtype=torch.float32, device=dev)
    path = resolve_path(kw["path"])
    with torch.cuda.device(dev):
        hl, dl = _lane_copies(lanes, dev)
        ws, wsb = _workspace(getattr(L, spec.pool_ws)(A, T_max, *spec.geometry(kw), *spec.ws_tail(kw, path)), dev)
        rc = getattr(L, spec.pool)(
            _ptr(pool.ring), _ptr(hl), _ptr(dl), len(lanes), A, _ptr(xs), dt, pool.slots, n, pitch, *spec.tail(kw),
            _ptr(out), T_max, _ptr(ws), wsb, path, _stream(dev))
    return _chunk_result(rc, out, spec.pool)


def stft_pool_forward(pool, lanes, x, A, T_max, wcos, wsin, packed, n_fft, hop, center, pad_mode, out_format,
                      sqrt_eps, path=None):
    return _pool("stft_forward", pool, lanes, x, A, T_max, locals())


def stft_filterbank_pool_forward(pool, lanes, x, A, T_max, wcos, wsin, packed, n_fft, hop, center, pad_mode,
                                 sqrt_eps, power, fb, fb_table=None, path=None):
    return _pool("stft_filterbank_forward", pool, lanes, x, A, T_max, locals())


def mfcc_pool_forward(pool, lanes, x, A, T_max, wcos, wsin, packed, n_fft, hop, center, pad_mode, sqrt_eps, power,
                      mel_basis, amin, ref, top_db, dct, fb_table=None, path=None):
    return _pool("mfcc_forward", pool, lanes, x, A, T_max, locals())


def cqt1992v2_pool_forward(pool, lanes, x, A, T_max, k_real, k_imag, packed, k_begin, k_end, hop, center, pad_mode,
                           scale, scale_all, out_format, sqrt_eps, path=None):
    return _pool("cqt1992v2_forward", pool, lanes, x, A, T_max, locals())


def cqt_pyramid_chunk_state_bytes(B: int, widths, hop: int, early_factor: int) -> int:
    w = (c_int32 * len(widths))(*[int(v) for v in widths])
    return int(lib().nnab_cqt_pyramid_chunk_state_bytes(int(B), len(widths), w, int(hop), int(early_factor)))


def cqt_pyramid_chunk_plan(received, n_carry, frames, n, flush, widths, hop, pad_mode, early_factor=1):
    """Host-only plan of one push (``nnab_debug_pyramid_chunk_plan``): per signal (R before, R after, ring
    length, first sample kept, FIR source origin, first FIR row or -1, head edge-fix end, tail edge-fix start),
    and the frame bound after the push.  Raises on counters no stream can have."""
    n_sig = len(widths) + (1 if early_factor > 1 else 0)
    w = (c_int32 * len(widths))(*[int(v) for v in widths])
    buf = (c_int64 * (8 * n_sig + 1))()
    _check(lib().nnab_debug_pyramid_chunk_plan(int(received), int(n_carry), int(frames), int(n), int(flush),
                                               len(widths), w, int(hop), int(early_factor), int(pad_mode), buf),
          "nnab_debug_pyramid_chunk_plan")
    return [tuple(buf[8 * s:8 * s + 8]) for s in range(n_sig)], int(buf[8 * n_sig])


def cqt_pyramid_chunk_forward(st, x, flush, T, banks_real, banks_imag, packed, lowpass, lowpass_packed,
                              early_filter, early_packed, early_factor, hop, pad_mode, n_bins, scale, scale_all,
                              out_format, sqrt_eps, path=None):
    """One push of ``nnaudio_b200.streaming.StreamingPyramid`` (``st``: its rings and counters); the remaining
    arguments are ``cqt_pyramid_forward``'s.  None when the configuration has no streamed plan
    (NNAB_EUNSUPPORTED, nothing enqueued)."""
    L = lib()
    xs, n, pitch, dt = _chunk_args(st, x)
    B, dev = st.batch, st.ring.device
    n_oct = len(banks_real)
    re_arr, im_arr, pk_arr, widths = _bank_arrays(banks_real, banks_imag, packed)
    out = torch.empty(_complex_shape(B, n_bins, T, out_format != FMT_MAGNITUDE), dtype=torch.float32, device=dev)
    path = resolve_path(path)
    with torch.cuda.device(dev):
        ws, wsb = _workspace(L.nnab_cqt_pyramid_chunk_workspace_bytes(
            B, st.received, st.n_carry, st.frames, n, int(flush), n_oct, widths, hop, early_factor, pad_mode), dev)
        rc = L.nnab_cqt_pyramid_chunk_forward(
            _ptr(st.ring), st.received, st.n_carry, st.frames, _ptr(xs), dt, B, n, pitch, int(flush), n_oct,
            re_arr, im_arr, pk_arr, widths, banks_real[0].shape[0], _ptr(lowpass), _ptr(lowpass_packed),
            _ptr(early_filter), _ptr(early_packed), early_factor, hop, pad_mode, n_bins, _ptr(scale), scale_all,
            out_format, sqrt_eps, _ptr(out) if T > 0 else None, T, _ptr(ws), wsb, path, _stream(dev))
    return _chunk_result(rc, out, "nnab_cqt_pyramid_chunk_forward")


def _lane_table(lanes):
    """A C copy of an (n_lanes, 6) int64 lane table (host-only calls)."""
    a = np.ascontiguousarray(np.asarray(lanes, dtype=np.int64).reshape(-1, 6))
    return a, (a.ctypes.data_as(c_void_p) if len(a) else None)


def cqt_pyramid_pool_plan(lanes, A, widths, hop, pad_mode, early_factor=1):
    """Host-only plan of one pool push (``nnab_debug_pyramid_pool_plan``): for each lane, the levels and frame
    bound of ``cqt_pyramid_chunk_plan``.  Raises on a lane table the library refuses."""
    n_sig = len(widths) + (1 if early_factor > 1 else 0)
    a, ptr = _lane_table(lanes)
    w = (c_int32 * len(widths))(*[int(v) for v in widths])
    buf = (c_int64 * max(1, len(a) * (8 * n_sig + 1)))()
    _check(lib().nnab_debug_pyramid_pool_plan(ptr, len(a), int(A), len(widths), w, int(hop), int(early_factor),
                                              int(pad_mode), buf), "nnab_debug_pyramid_pool_plan")
    out = []
    for i in range(len(a)):
        o = buf[i * (8 * n_sig + 1):(i + 1) * (8 * n_sig + 1)]
        out.append(([tuple(o[8 * s:8 * s + 8]) for s in range(n_sig)], int(o[8 * n_sig])))
    return out


def cqt_pyramid_pool_workspace_bytes(lanes, A, T_max, widths, hop, early_factor, pad_mode) -> int:
    a, ptr = _lane_table(lanes)
    w = (c_int32 * len(widths))(*[int(v) for v in widths])
    return int(lib().nnab_cqt_pyramid_pool_workspace_bytes(ptr, len(a), int(A), int(T_max), len(widths), w,
                                                            int(hop), int(early_factor), int(pad_mode)))


def cqt_pyramid_pool_forward(pool, lanes, x, A, T_max, banks_real, banks_imag, packed, lowpass, lowpass_packed,
                             early_filter, early_packed, early_factor, hop, pad_mode, n_bins, scale, scale_all,
                             out_format, sqrt_eps, path=None):
    """One push of ``nnaudio_b200.streaming.PyramidPool``: ``lanes`` its (n_lanes, 6) lane table (the A lanes with
    frames first), ``x`` the (slots, n) chunk; ``pool`` carries the rings (``pool.ring``) and ``pool.slots``.  The
    remaining arguments are ``cqt_pyramid_forward``'s.  Returns the (A, n_bins, T_max[, 2]) frames, or None when the configuration has no streamed plan (NNAB_EUNSUPPORTED, nothing enqueued)."""
    L = lib()
    xs, n, pitch, dt = _chunk_args(pool, x)
    dev = pool.ring.device
    out = torch.empty(_complex_shape(A, n_bins, T_max, out_format != FMT_MAGNITUDE), dtype=torch.float32, device=dev)
    n_oct = len(banks_real)
    re_arr, im_arr, pk_arr, widths = _bank_arrays(banks_real, banks_imag, packed)
    path = resolve_path(path)
    with torch.cuda.device(dev):
        ws, wsb = _workspace(cqt_pyramid_pool_workspace_bytes(lanes, A, T_max, widths, hop, early_factor, pad_mode),
                             dev)
        hl, dl = _lane_copies(lanes, dev)
        rc = L.nnab_cqt_pyramid_pool_forward(
            _ptr(pool.ring), _ptr(hl), _ptr(dl), len(lanes), A, _ptr(xs), dt, pool.slots, n, pitch, n_oct, re_arr,
            im_arr, pk_arr, widths, banks_real[0].shape[0], _ptr(lowpass), _ptr(lowpass_packed),
            _ptr(early_filter), _ptr(early_packed), early_factor, hop, pad_mode, n_bins, _ptr(scale), scale_all,
            out_format, sqrt_eps, _ptr(out) if out.numel() else None, T_max, _ptr(ws), wsb, path, _stream(dev))
    return _chunk_result(rc, out, "nnab_cqt_pyramid_pool_forward")


def istft_chunk_forward(st, X, flush, length, n_out, packed, window, n_fft, hop, center):
    """One push of a streamed inverse STFT: X (B, f_in, T, 2) fp32 CUDA (T may be 0) -> the n_out samples it
    completes.  ``st``: device state ``st.state`` and host counters ``st.frames`` / ``st.emitted``."""
    L = lib()
    X = _dev_f32(X, "X")
    X = X if X.is_contiguous() else X.contiguous()
    B, f_in, T, _ = X.shape
    dev = st.state.device
    out = torch.empty((B, n_out), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        ws, wsb = _workspace(L.nnab_istft_chunk_workspace_bytes(B, f_in, T, n_fft, hop), dev)
        rc = L.nnab_istft_chunk_forward(_ptr(st.state), st.frames, st.emitted, _ptr(X) if T > 0 else None, B,
                                        f_in, T, _ptr(packed), _ptr(window), n_fft, hop, int(center), int(flush),
                                        -1 if length is None else int(length), _ptr(out), n_out, _ptr(ws), wsb,
                                        _stream(dev))
    _check(rc, "nnab_istft_chunk_forward")
    return out


ISTFT_LANE_FIELDS = ("slot", "row", "frames", "emitted", "T", "end", "length")


def istft_pool_forward(pool, lanes, X, A, n_max, T_max, packed, window, n_fft, hop, center):
    """One push of an inverse STFT pool (nnaudio_b200.streaming.InversePool): ``lanes`` is the push's (n_lanes, 7)
    int64 table of nnab_istft_lane rows (the A lanes with samples first), X the (R, f_in, t, 2) fp32 CUDA frames.
    ``pool`` carries the device state ``pool.state`` (one row per slot) and ``pool.slots``.  Returns the (A, n_max)
    samples, zeros past each row's count."""
    L = lib()
    dev = pool.state.device
    out = torch.empty((A, n_max), dtype=torch.float32, device=dev)
    if len(lanes) == 0:
        return out
    X = _dev_f32(X, "X")
    X = X if X.is_contiguous() else X.contiguous()
    R, f_in, t, _ = X.shape
    with torch.cuda.device(dev):
        hl, dl = _lane_copies(lanes, dev)
        ws, wsb = _workspace(L.nnab_istft_pool_workspace_bytes(len(lanes), f_in, T_max, n_fft, hop), dev)
        rc = L.nnab_istft_pool_forward(
            _ptr(pool.state), _ptr(hl), _ptr(dl), len(lanes), A, pool.slots, _ptr(X) if X.numel() else None, R,
            f_in, t, _ptr(packed), _ptr(window), n_fft, hop, int(center), _ptr(out) if out.numel() else None, n_max,
            T_max, _ptr(ws), wsb, _stream(dev))
    _check(rc, "nnab_istft_pool_forward")
    return out


# --------------------------------------------------------------------------- #
# device pools (nnaudio_b200.streaming.DeviceStreamPool / DeviceInversePool): every per-push number on the device.
# The arguments that do not change from push to push (module buffers, outputs, workspace) are bound once.
# --------------------------------------------------------------------------- #
LANE_OK, LANE_ELENGTH, LANE_EENDED, LANE_ESHORT, LANE_ENOFRAMES, LANE_ELENGTH_SHORT = range(6)


def pool_frame_cap(chunk: int, K: int, hop: int, pad: int, pad_mode: int) -> int:
    """The most frames one push of at most ``chunk`` samples can return, an end included."""
    return int(lib().nnab_pool_frame_cap(int(chunk), int(K), int(hop), int(pad), int(pad_mode)))


def istft_pool_sample_cap(frames: int, n_fft: int, hop: int, center: bool) -> int:
    """The most samples one inverse push of at most ``frames`` frames can return, a flush included."""
    return int(lib().nnab_istft_pool_sample_cap(int(frames), int(n_fft), int(hop), int(center)))


def pool_device_bind(name, kw, slots, T_cap, device, path=None):
    """The fixed part of a device pool's pushes on the offline call ``name`` with arguments ``kw``: returns
    (C function, output (slots, ..., T_cap), workspace, argument tail after the chunk pitch, stream excluded)."""
    if name not in _SPECS:
        raise ValueError(f"no device pool for {name}")
    spec, L = _SPECS[name], lib()
    path = resolve_path(path)
    out = torch.zeros(spec.shape(slots, T_cap, kw), dtype=torch.float32, device=device)
    ws, wsb = _workspace(getattr(L, spec.pool_ws)(slots, T_cap, *spec.geometry(kw), *spec.ws_tail(kw, path)), device)
    return getattr(L, spec.device), out, ws, spec.tail(kw) + (_ptr(out), T_cap, _ptr(ws), wsb, path)


def pool_device_forward(pool, x, lengths, end):
    """One push of a DeviceStreamPool (``pool``: its device buffers and bound call); every argument checked by the
    caller.  False when the plan cannot read the chunk (NNAB_EUNSUPPORTED)."""
    dev = pool.ring.device
    with torch.cuda.device(dev):
        rc = pool._fn(_ptr(pool.ring), _ptr(pool.counters), _ptr(lengths), _ptr(end), _ptr(pool.errors),
                      _ptr(pool.error_info), _ptr(pool.counts), _ptr(pool._lanes), _ptr(x), _WAVE_DTYPES[x.dtype],
                      pool.slots, x.shape[1], x.stride(0) if x.shape[0] > 1 else x.shape[1], *pool._tail,
                      _stream(dev))
    if rc == EUNSUPPORTED:
        return False
    _check(rc, pool._fn.__name__)
    return True


def istft_pool_device_forward(pool, X, counts, end, length):
    """One push of a DeviceInversePool; every argument checked by the caller."""
    dev = pool.state.device
    with torch.cuda.device(dev):
        rc = lib().nnab_istft_pool_device_forward(
            _ptr(pool.state), _ptr(pool.counters), _ptr(counts), _ptr(end), _ptr(length), _ptr(pool.errors),
            _ptr(pool.error_info), _ptr(pool.counts), _ptr(pool._lanes), pool.slots, _ptr(X), pool.f_in,
            pool.frames_cap, _ptr(pool._packed), _ptr(pool._window), pool.n_fft, pool.hop, int(pool.center),
            _ptr(pool.samples), pool.n_cap, _ptr(pool._ws), pool._ws.numel(), _stream(dev))
    _check(rc, "nnab_istft_pool_device_forward")


def pool_device_reset(pool, mask):
    """Zero the counters, errors and error values of the slots where ``mask`` (uint8 CUDA, or None: all) is set."""
    dev = pool.counters.device
    with torch.cuda.device(dev):
        _check(lib().nnab_pool_device_reset(_ptr(pool.counters), _ptr(pool.errors), _ptr(pool.error_info), _ptr(mask),
                                            pool.slots, _stream(dev)), "nnab_pool_device_reset")


def debug_device_pool_plan(counters, lengths, end, errors, error_info, n, K, hop, pad, pad_mode):
    """Host-only run of a device pool's plan launch (``nnab_debug_device_pool_plan``) on numpy arrays: counters
    (3, slots) int64, errors (slots,) int32 and error_info (slots, 2) int64 are updated in place; returns (lanes
    (slots, 6) int64, counts (slots,) int32)."""
    slots = len(lengths)
    lengths = np.ascontiguousarray(lengths, np.int32)
    end = np.ascontiguousarray(end, np.uint8)
    lanes = np.zeros((slots, 6), np.int64)
    counts = np.zeros(slots, np.int32)
    p = lambda a: a.ctypes.data_as(c_void_p)
    _check(lib().nnab_debug_device_pool_plan(p(counters), p(lengths), p(end), p(errors), p(error_info), p(counts),
                                             p(lanes), slots, int(n), int(K), int(hop), int(pad), int(pad_mode)),
           "nnab_debug_device_pool_plan")
    return lanes, counts


def debug_device_istft_plan(counters, frame_counts, end, length, errors, error_info, t, n_fft, hop, center):
    """``debug_device_pool_plan`` for a device inverse pool: returns (lanes (slots, 7) int64, counts (slots,))."""
    slots = len(frame_counts)
    frame_counts = np.ascontiguousarray(frame_counts, np.int32)
    end = np.ascontiguousarray(end, np.uint8)
    length = np.ascontiguousarray(length, np.int64)
    lanes = np.zeros((slots, 7), np.int64)
    counts = np.zeros(slots, np.int32)
    p = lambda a: a.ctypes.data_as(c_void_p)
    _check(lib().nnab_debug_device_istft_plan(p(counters), p(frame_counts), p(end), p(length), p(errors),
                                              p(error_info), p(counts), p(lanes), slots, int(t), int(n_fft), int(hop),
                                              int(center)), "nnab_debug_device_istft_plan")
    return lanes, counts


def _widths(widths):
    return (c_int32 * len(widths))(*[int(v) for v in widths])


def cqt_pyramid_pool_device_caps(chunk, widths, hop, early_factor, pad_mode):
    """The fixed geometry of a device pyramid pool (``nnab_cqt_pyramid_pool_device_caps``, host only): (T_cap, the
    most FIR outputs per lane of each stage (0 for the last signal), the most samples one push stores into each
    signal's ring).  Raises if a push without an end could be refused."""
    n_sig = len(widths) + (1 if early_factor > 1 else 0)
    buf = (c_int64 * (1 + 2 * n_sig))()
    _check(lib().nnab_cqt_pyramid_pool_device_caps(int(chunk), len(widths), _widths(widths), int(hop),
                                                   int(early_factor), int(pad_mode), buf),
           "nnab_cqt_pyramid_pool_device_caps")
    return int(buf[0]), list(buf[1:1 + n_sig]), list(buf[1 + n_sig:1 + 2 * n_sig])


def pyramid_pool_device_bind(kw, slots, chunk, T_cap, device, path=None):
    """``pool_device_bind`` for a device pyramid pool on the pyramid arguments ``kw`` (``cqt_pyramid_forward``'s):
    (C function, output (slots, n_bins, T_cap[, 2]), workspace, argument tail after the chunk pitch).  The tail holds
    the ctypes bank arrays; the caller keeps the tensors of ``kw`` alive."""
    L = lib()
    path = resolve_path(path)
    re_arr, im_arr, pk_arr, widths = _bank_arrays(kw["banks_real"], kw["banks_imag"], kw["packed"])
    n_oct = len(kw["banks_real"])
    out = torch.zeros(_complex_shape(slots, kw["n_bins"], T_cap, kw["out_format"] != FMT_MAGNITUDE),
                      dtype=torch.float32, device=device)
    ws, wsb = _workspace(L.nnab_cqt_pyramid_pool_device_workspace_bytes(
        slots, chunk, n_oct, widths, kw["hop"], kw["early_factor"], kw["pad_mode"]), device)
    tail = (n_oct, re_arr, im_arr, pk_arr, widths, kw["banks_real"][0].shape[0], _ptr(kw["lowpass"]),
            _ptr(kw["lowpass_packed"]), _ptr(kw["early_filter"]), _ptr(kw["early_packed"]), kw["early_factor"],
            kw["hop"], kw["pad_mode"], kw["n_bins"], _ptr(kw["scale"]), kw["scale_all"], kw["out_format"],
            kw["sqrt_eps"], _ptr(out), T_cap, _ptr(ws), wsb, path)
    return L.nnab_cqt_pyramid_pool_device_forward, out, ws, tail


def debug_device_pyramid_plan(counters, lengths, end, errors, error_info, n, widths, hop, early_factor, pad_mode):
    """``debug_device_pool_plan`` for a device pyramid pool (``nnab_debug_device_pyramid_plan``): returns (lanes
    (slots, 6) int64, counts (slots,) int32)."""
    slots = len(lengths)
    lengths = np.ascontiguousarray(lengths, np.int32)
    end = np.ascontiguousarray(end, np.uint8)
    lanes = np.zeros((slots, 6), np.int64)
    counts = np.zeros(slots, np.int32)
    p = lambda a: a.ctypes.data_as(c_void_p)
    _check(lib().nnab_debug_device_pyramid_plan(p(counters), p(lengths), p(end), p(errors), p(error_info), p(counts),
                                                p(lanes), slots, int(n), len(widths), _widths(widths), int(hop),
                                                int(early_factor), int(pad_mode)), "nnab_debug_device_pyramid_plan")
    return lanes, counts


# The overlap-add GEMM of the inverse STFT and of both gradients takes frames of at most this many output samples
# (n_fft of the inverse, kernel width of the gradients): 128 N tiles of 256.
OLA_MAX_WIDTH = 32768


def ola_plan(F_out: int, K_gemm: int, M_rows: int, k_splits_hint: int = 0) -> dict:
    """Host-only launch shape of the overlap-add GEMM (``nnab_debug_ola_plan``; the operands of each caller are
    listed in include/nnab.h)."""
    out = (ctypes.c_double * 5)()
    _check(lib().nnab_debug_ola_plan(int(F_out), int(K_gemm), int(M_rows), int(k_splits_hint), out),
           "nnab_debug_ola_plan")
    return dict(supported=bool(out[0]), bn=int(out[1]), n_tiles=int(out[2]), k_splits=int(out[3]),
                exec_flops=float(out[4]))


def _check_ola(rc: int, what: str, width: int, name: str):
    """``_check`` for the overlap-add GEMM's callers: a frame wider than the GEMM takes is named as such."""
    if rc == EUNSUPPORTED and width > OLA_MAX_WIDTH:
        raise RuntimeError(f"{what} failed: {name} {width} is above the overlap-add GEMM's limit of "
                           f"{OLA_MAX_WIDTH} samples (status {rc})")
    _check(rc, what)


def pack_istft_basis(kernel_cos: torch.Tensor, kernel_sin: torch.Tensor, f_in: int, onesided: bool):
    """Tensor-core packing of the (n_fft, n_fft) inverse kernels; the mirroring of a
    one-sided spectrum (utils.py:63-70) is folded into the packed rows."""
    L = lib()
    n_fft = kernel_cos.shape[0]
    packed = torch.empty(L.nnab_packed_istft_bytes(n_fft, f_in), dtype=torch.uint8,
                         device=kernel_cos.device)
    with torch.cuda.device(kernel_cos.device):
        _check(L.nnab_pack_istft_basis(_ptr(kernel_cos), _ptr(kernel_sin), n_fft, f_in,
                                       int(onesided), _ptr(packed), _stream(kernel_cos.device)),
               "nnab_pack_istft_basis")
    return packed


def istft_forward(X, packed, window, n_fft, hop, center, length):
    """X (B, f_in, T, 2) fp32 CUDA -> waveform (B, out_len)."""
    if X.dim() == 4 and X.shape[0] > MAX_BATCH:
        return torch.cat([istft_forward(X[i:i + MAX_BATCH], packed, window, n_fft, hop, center, length)
                          for i in _batch_starts(X.shape[0])], 0)
    L = lib()
    X = _dev_f32(X, "X")
    X = X if X.is_contiguous() else X.contiguous()
    B, f_in, T, _ = X.shape
    ola_len = n_fft + hop * (T - 1)
    pad = n_fft // 2
    offset = pad if center else 0
    want = length if length is not None else (ola_len - 2 * pad if center else ola_len)
    want = max(0, min(want, ola_len - offset))
    out = torch.empty((B, want), dtype=torch.float32, device=X.device)
    with torch.cuda.device(X.device):
        ws, wsb = _workspace(L.nnab_istft_workspace_bytes(B, f_in, T, n_fft, hop), X.device)
        rc = L.nnab_istft_forward(_ptr(X), B, f_in, T, _ptr(packed), _ptr(window), n_fft, hop,
                                  int(center), -1 if length is None else int(length), _ptr(out),
                                  want, _ptr(ws), wsb, _stream(X.device))
    _check_ola(rc, "nnab_istft_forward", n_fft, "n_fft")
    return out


def fir_decimate(x, fir, factor):
    """EXPERIMENTAL: y = conv1d(x, fir, stride=factor, padding=(taps-1)//2) for (B, L) rows."""
    if x.dim() == 2 and x.shape[0] > MAX_BATCH:
        return torch.cat([fir_decimate(x[i:i + MAX_BATCH], fir, factor) for i in _batch_starts(x.shape[0])], 0)
    L = lib()
    x, B, Ln, pitch = _rows(x)
    fir = _dev_f32(fir, "fir").reshape(-1).contiguous()
    taps = fir.numel()
    half = (taps - 1) // 2
    Ly = (Ln + 2 * half - taps) // factor + 1
    y = torch.empty((B, Ly), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _check(L.nnab_fir_decimate(_ptr(x), B, Ln, pitch, _ptr(fir), taps, int(factor), _ptr(y), Ly,
                                   _stream(x.device)), "nnab_fir_decimate")
    return y


def fir_decimate_adjoint(g, fir, factor, L_in):
    """EXPERIMENTAL: gradient of fir_decimate w.r.t. its input, (B, Ly) -> (B, L_in)."""
    if g.dim() == 2 and g.shape[0] > MAX_BATCH:
        return torch.cat([fir_decimate_adjoint(g[i:i + MAX_BATCH], fir, factor, L_in)
                          for i in _batch_starts(g.shape[0])], 0)
    L = lib()
    g, B, Ly, pitch = _rows(g)
    fir = _dev_f32(fir, "fir").reshape(-1).contiguous()
    dx = torch.empty((B, L_in), dtype=torch.float32, device=g.device)
    with torch.cuda.device(g.device):
        _check(L.nnab_fir_decimate_adjoint(_ptr(g), B, Ly, pitch, _ptr(fir), fir.numel(), int(factor),
                                           _ptr(dx), int(L_in), _stream(g.device)),
               "nnab_fir_decimate_adjoint")
    return dx


def pack_adjoint_basis(w_re: torch.Tensor, w_im: torch.Tensor):
    """W^T packing of an (F, K) forward basis pair for the input-gradient GEMM."""
    L = lib()
    F, K = w_re.shape
    packed = torch.empty(L.nnab_packed_adjoint_bytes(K, F), dtype=torch.uint8, device=w_re.device)
    with torch.cuda.device(w_re.device):
        _check(L.nnab_pack_adjoint_basis(_ptr(w_re), _ptr(w_im), F, K, _ptr(packed),
                                         _stream(w_re.device)), "nnab_pack_adjoint_basis")
    return packed


def framed_backward_input(g, packed_adj, K, hop, center, pad_mode, L_in):
    """g (B, F, T, 2) -> dx (B, L_in)."""
    if g.dim() == 4 and g.shape[0] > MAX_BATCH:
        return torch.cat([framed_backward_input(g[i:i + MAX_BATCH], packed_adj, K, hop, center, pad_mode, L_in)
                          for i in _batch_starts(g.shape[0])], 0)
    L = lib()
    g = _dev_f32(g, "grad")
    g = g if g.is_contiguous() else g.contiguous()
    B, F, T, _ = g.shape
    dx = torch.empty((B, L_in), dtype=torch.float32, device=g.device)
    with torch.cuda.device(g.device):
        ws, wsb = _workspace(
            L.nnab_framed_backward_input_workspace_bytes(B, L_in, K, F, hop, int(center)), g.device)
        rc = L.nnab_framed_backward_input(_ptr(g), B, F, T, _ptr(packed_adj), K, hop, int(center),
                                          pad_mode, _ptr(dx), L_in, _ptr(ws), wsb,
                                          _stream(g.device))
    _check_ola(rc, "nnab_framed_backward_input", K, "kernel width")
    return dx


def framed_backward_weight(g, x, K, hop, center, pad_mode):
    """g (B, F, T, 2), x (B, L) -> (d w_re, d w_im), each (F, K).  The clips are the GEMM's K, so a batch of
    more than ``MAX_BATCH`` clips is the sum of its chunks' gradients, added in chunk order."""
    if g.dim() == 4 and g.shape[0] > MAX_BATCH:
        d_re = d_im = None
        for i in _batch_starts(g.shape[0]):
            r, m = framed_backward_weight(g[i:i + MAX_BATCH], x[i:i + MAX_BATCH], K, hop, center, pad_mode)
            d_re, d_im = (r, m) if d_re is None else (d_re + r, d_im + m)
        return d_re, d_im
    L = lib()
    g = _dev_f32(g, "grad")
    g = g if g.is_contiguous() else g.contiguous()
    x, B, Ln, pitch = _rows(x)
    _, F, T, _ = g.shape
    dw = torch.empty((2 * F, K), dtype=torch.float32, device=g.device)
    with torch.cuda.device(g.device):
        ws, wsb = _workspace(
            L.nnab_framed_backward_weight_workspace_bytes(B, Ln, K, F, hop, int(center)), g.device)
        rc = L.nnab_framed_backward_weight(_ptr(g), _ptr(x), B, Ln, pitch, F, T, K, hop,
                                           int(center), pad_mode, _ptr(dw), _ptr(ws), wsb,
                                           _stream(g.device))
    _check_ola(rc, "nnab_framed_backward_weight", K, "kernel width")
    return dw[:F], -dw[F:]


# --------------------------------------------------------------------------- #
# PCEN (nnaudio_b200.pcen): one (B, C, T) spectrogram per call; the parameters are (1,) or (C,) fp32 CUDA tensors
# --------------------------------------------------------------------------- #
SIGNATURES["nnab_pcen_forward"] = (
    c_int, [_P, c_int64, c_int, c_int64, _P, _P, _P, _P, c_int, c_float, _P, _P, _P, _P, c_int64, _P, _P, _P])
SIGNATURES["nnab_pcen_workspace_bytes"] = (c_size_t, [c_int64, c_int])
SIGNATURES["nnab_pcen_backward"] = (
    c_int, [_P, _P, _P, c_int64, c_int, c_int64, _P, _P, _P, _P, c_int, c_float, _P, _P, _P, c_size_t, _P])
SIGNATURES["nnab_pcen_reset"] = (c_int, [_P, _P, c_int64, c_int, _P])


def _pcen_params(params):
    """(four pointers, parameter stride) of the (s, gain, bias, power) tensors: one value each, or one per channel."""
    stride = 1 if params[0].numel() > 1 else 0
    return [_ptr(p) for p in params], stride


def pcen_forward(E, params, eps, M=None, stream_state=None, row_slot=None, counts=None):
    """E (B, C, T) contiguous fp32 CUDA -> P (B, C, T).  ``M``: the training call's (B, C, T) smoother output.
    ``stream_state``: (state (slots, C) fp32, primed (slots, C) uint8) of a streamed call, with the int32 device
    ``row_slot`` (B,) / ``counts`` (B,) or None.  Every argument checked by the caller."""
    B, C, T = E.shape
    P = _new_out((B, C, T), E.device)
    (s, gain, bias, power), stride = _pcen_params(params)
    state, primed = stream_state if stream_state is not None else (None, None)
    with torch.cuda.device(E.device):
        rc = lib().nnab_pcen_forward(_ptr(E), B, C, T, s, gain, bias, power, stride, float(eps), _ptr(P), _ptr(M),
                                     _ptr(state), _ptr(primed), 0 if state is None else state.shape[0],
                                     _ptr(row_slot), _ptr(counts), _stream(E.device))
    _check(rc, "nnab_pcen_forward")
    return P


def pcen_backward(E, M, gP, params, eps, want_E=True, want_params=True):
    """(grad_E (B, C, T) or None, grad_params (4, n) or None) of the training call on E, its M and grad_P;
    ``n`` is C for per-channel parameters, else 1 (rows s, gain, bias, power)."""
    L = lib()
    B, C, T = E.shape
    (s, gain, bias, power), stride = _pcen_params(params)
    dE = torch.empty((B, C, T), dtype=torch.float32, device=E.device) if want_E else None
    dp = torch.empty((4, C if stride else 1), dtype=torch.float32, device=E.device) if want_params else None
    with torch.cuda.device(E.device):
        ws, wsb = _workspace(L.nnab_pcen_workspace_bytes(B, C) if want_params else 0, E.device)
        rc = L.nnab_pcen_backward(_ptr(E), _ptr(M), _ptr(gP), B, C, T, s, gain, bias, power, stride, float(eps),
                                  _ptr(dE), _ptr(dp), _ptr(ws), wsb, _stream(E.device))
    _check(rc, "nnab_pcen_backward")
    return dE, dp


def pcen_reset(primed, mask):
    """Un-prime the (slots, C) stream state where the uint8 device ``mask`` (slots,) is set (None: every slot)."""
    with torch.cuda.device(primed.device):
        _check(lib().nnab_pcen_reset(_ptr(primed), _ptr(mask), primed.shape[0], primed.shape[1],
                                     _stream(primed.device)), "nnab_pcen_reset")
