"""The four-phase block-partial STFT kernel with separate MMA and epilogue warps (csrc/tcb_kernels.cu,
framed_tcb_ws_kernel; -m gpu).  Its MMA warps run the K loop of a CTA's next tile and refill the stage ring while
its epilogue warps drain the current tile, handing the one accumulator tile back and forth through two
mbarriers.  Grids of 1, 2, 3 and all SMs (an SM reserve) give CTAs many tiles each, one tile, or two; every
accumulator sees the same wgmma sequence and every (family, tile) the same epilogue, so outputs must be bitwise
equal across grids and across two identical calls.  The executed-MMA-flop counter proves the four-phase instance
ran, at a tile width this kernel takes (nb <= 88)."""
import warnings

import numpy as np
import pytest
import torch

import block_domain as bd
from helpers import build, rel_errors, run_oracle
from nnaudio_b200 import _C

pytestmark = pytest.mark.gpu

WS_NB_MAX = 88  # TCB_WS_NB_MAX

# (class, constructor, route): hop % 128 == 0 everywhere (four phases); the launch takes this kernel for the
# fused filterbank and the operand planes
CONFIGS = {
    "mel_fast": ("MelSpectrogram", dict(sr=16000, n_fft=512, hop_length=128, n_mels=40), "fast"),
    # power != 2: the rolled MelRun epilogue (its atomic adds may reorder: held to the oracle, not bitwise)
    "mel_rolled": ("MelSpectrogram", dict(sr=16000, n_fft=512, hop_length=128, n_mels=40, power=1.0), "rolled"),
    "gammatone_planes": ("Gammatonegram", dict(sr=22050, n_fft=2048, hop_length=512, n_bins=64), "planes"),
}


def _nb(cls, ctor, mod):
    n_fft, hop = ctor["n_fft"], ctor["hop_length"]
    if cls == "MelSpectrogram":
        return bd.fbank_nb(mod.mel_basis.detach().cpu().numpy(), n_fft, hop)[0]
    return bd.bp.choose_nb(bd.basis_bins(n_fft, hop))


def _length(n_fft, hop, m_tiles):
    """Clip length whose centred block rows fill exactly m_tiles four-phase M tiles (33 - R rows each)."""
    R = n_fft // hop
    return m_tiles * (33 - R) * hop - n_fft


def _run(mod, x, reserve):
    """(mod(x), executed MMA flops, persistent-grid ledger) of one call under an SM reserve of ``reserve``."""
    old = _C.set_sm_reserve(reserve)
    _C.persistent_grid_read()
    _C.profile_read_exec_flops()
    _C.profile_enable(True)
    try:
        with torch.no_grad(), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            y = mod(x)
        torch.cuda.synchronize()
    finally:
        _C.profile_enable(False)
        _C.profile_read()
        _C.set_sm_reserve(old)
    return y, _C.profile_read_exec_flops(), _C.persistent_grid_read()


@pytest.mark.parametrize("tiles_vs_sms", [-1, 0, 1])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_ws_kernel_grids_bitwise(name, tiles_vs_sms):
    cls, ctor, route = CONFIGS[name]
    n_fft, hop = ctor["n_fft"], ctor["hop_length"]
    mod = build(cls, ctor).cuda()
    nb = _nb(cls, ctor, mod)
    assert nb <= WS_NB_MAX, (name, nb)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_tiles = bd.bp.n_tiles_of(bd.basis_bins(n_fft, hop), nb)
    # tiles below, equal to, just above one per SM (rounded up to whole M tiles)
    m_tiles = -(-(sms + tiles_vs_sms) // n_tiles)
    L = _length(n_fft, hop, m_tiles)
    assert bd.geometry(n_fft, hop, 1, L, True)[2] == m_tiles
    xn = np.random.RandomState(11 + tiles_vs_sms).standard_normal((1, L)).astype(np.float32)
    x = torch.from_numpy(xn).cuda()

    want_flops = bd.block_exec_flops(n_fft, hop, 1, L, True, nb=nb)
    outs = []
    for grid in (sms, 1, 2, 3):
        y, flops, ledger = _run(mod, x, sms - grid)
        if grid < sms:  # each persistent launch (the block kernel, and the planes GEMM) ran at this grid
            n = ledger[0]
            assert n >= 1 and ledger == (n, n * grid, grid, grid), (name, grid, ledger)
        want = want_flops
        if route == "planes":
            want += bd.planes_gemm_flops(n_fft, hop, 1, y.shape[-1], mod.gammatone_basis.shape[0])
        assert flops == want, (name, grid, flops, want)
        outs.append((grid, y))
    ref = outs[0][1]
    if route == "rolled":
        want = run_oracle(cls, mod, xn, {})
        for grid, y in outs:
            emax, el2 = rel_errors(y.cpu().numpy(), want)
            assert emax < 1e-4 and el2 < 1e-4, (name, grid, emax, el2)
        return
    for grid, y in outs[1:]:
        assert torch.equal(ref, y), (name, grid)
    again = _run(mod, x, 0)[0]
    assert torch.equal(ref, again), name
    emax, el2 = rel_errors(ref.cpu().numpy(), run_oracle(cls, mod, xn, {}))
    assert emax < 1e-4 and el2 < 1e-4, (name, emax, el2)
