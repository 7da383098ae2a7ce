"""No-GPU checks of the drop-in boundary: libnnab.so loads and exports every
symbol include/nnab.h declares; the ctypes table covers exactly that set."""
import ctypes
import os
import re

from helpers import ROOT

from nnaudio_b200 import _C


def _declared():
    text = open(os.path.join(ROOT, "include", "nnab.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(nnab_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    names = _declared()
    assert len(names) >= 15
    handle = ctypes.CDLL(_C.LIB_PATH)
    for n in names:
        assert hasattr(handle, n), f"libnnab.so does not export {n}"


def test_ctypes_table_matches_header():
    assert sorted(_C.SIGNATURES) == _declared()


def test_abi_version_and_strerror():
    lib = _C.lib()
    assert lib.nnab_abi_version() == 1
    assert lib.nnab_strerror(0) == b"ok"
    assert b"tensor-core" in lib.nnab_strerror(-2)
    assert lib.nnab_pack_tile_n(1025) == 208 and lib.nnab_pack_tile_n(84) == 176


def test_argument_validation_precedes_any_cuda_work():
    """Status codes for malformed calls are decided on the host, before a device is touched
    (so they are checkable here); a well-formed call on a GPU-less host reports a CUDA error
    instead of computing anything (no CPU fallback behind the C ABI either)."""
    lib = _C.lib()
    P = ctypes.c_void_p
    x = w = out = P(256)  # never dereferenced on the host
    EINVAL = -1

    def stft(hop=128, T=32, L=4000, pitch=4000, fmt=0, xp=x):
        return lib.nnab_stft_forward(xp, 4, L, pitch, w, w, None, 512, 257, hop, 1, 0, fmt, 0.0, out, T,
                                     None, 0, 0, None)

    assert stft(hop=0) == EINVAL
    assert stft(T=99) == EINVAL, "frame count must equal (L + 2*pad - n_fft) // hop + 1"
    assert stft(pitch=100) == EINVAL, "row pitch shorter than the clip"
    assert stft(fmt=7) == EINVAL
    assert stft(xp=None) == EINVAL
    assert stft(L=100) == EINVAL, "reflect padding needs pad < L (stft.py:283-286)"
    assert lib.nnab_istft_forward(None, 1, 257, 10, None, None, 512, 128, 1, -1, None, 0, None, 0,
                                  None) == EINVAL
    assert lib.nnab_framed_backward_input(None, 1, 257, 10, None, 512, 128, 1, 0, None, 1000, None, 0,
                                          None) == EINVAL
    assert lib.nnab_framed_backward_weight(None, None, 1, 1000, 1000, 257, 10, 512, 128, 1, 0, None,
                                           None, 0, None) == EINVAL
    import torch
    if not torch.cuda.is_available():
        rc = stft()
        assert rc in (-2, -4), rc  # NNAB_EARCH / NNAB_ECUDA — never NNAB_OK
        assert lib.nnab_strerror(rc) != b"ok"


def test_size_queries_are_host_only_and_consistent():
    lib = _C.lib()
    # cfg2: bf16 hi+lo planes of the padded batch (57 MB) and the packed basis (17 MB), DESIGN.md §2
    ws = lib.nnab_stft_workspace_bytes(64, 220500, 2048, 1025, 512, 1, 0)
    assert 56_000_000 < ws < 60_000_000
    assert lib.nnab_stft_workspace_bytes(64, 220500, 2048, 1025, 512, 1, 1) == 0, "SIMT path needs none"
    assert lib.nnab_packed_basis_bytes(1025, 2048) == 2 * 2 * 2080 * 2048
    assert lib.nnab_stft_workspace_bytes(128, 220500, 2048, 1025, 512, 1, 0) > ws
    assert lib.nnab_packed_fir_bytes(256, 2) > 0 and lib.nnab_packed_adjoint_bytes(2048, 1025) > 0
    assert lib.nnab_istft_workspace_bytes(4, 1025, 100, 2048, 512) > 0
    assert lib.nnab_framed_backward_input_workspace_bytes(4, 22050, 2048, 1025, 512, 1) > 0
    assert lib.nnab_framed_backward_weight_workspace_bytes(4, 22050, 2048, 1025, 512, 1) > 0
    assert lib.nnab_cqt_pyramid_workspace_bytes(4, 65536, 7, 1, 512, 512, 0) > 0
