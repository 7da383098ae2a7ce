"""Block-partial STFT kernel (csrc/tcb_kernels.cu) across grid sizes (-m gpu): the persistent CTAs share the
stage ring's refills with the epilogue of the previous tile, and a grid of one CTA (an SM reserve that leaves
one SM) runs every tile through the same ring back to back.  Every accumulator sees the same wgmma sequence
either way, so the outputs must be bitwise equal, including the masked rows of a partial last M tile.
Magnitude STFT (R = 4 and R = 2), the fused Mel epilogue and the Gammatone operand planes are checked, each
also against the CPU oracle."""
import warnings

import numpy as np
import pytest
import torch

from helpers import build, rel_errors, run_oracle
from nnaudio_b200 import _C

pytestmark = pytest.mark.gpu

# (class, constructor, input shape, forward kwargs): n_fft = 4 hop (116 frames per 128-row tile), lengths
# chosen for an odd number of M tiles: 3 x 83 block rows -> 3 tiles, 5 x 63 -> 3; n_fft = 2 hop (124 frames
# per tile): 276 -> 3
CONFIGS = {
    "stft_magnitude_odd_m": ("STFT", dict(n_fft=1024, hop_length=256, sr=16000, output_format="Magnitude"),
                             (3, 20000), {}),
    "mel_fused_odd_m": ("MelSpectrogram", dict(sr=16000, n_fft=1024, hop_length=256, n_mels=64), (3, 20000), {}),
    "gammatone_planes": ("Gammatonegram", dict(sr=22050, n_fft=2048, hop_length=512, n_bins=64), (5, 30000), {}),
    "stft_hop_half": ("STFT", dict(n_fft=512, hop_length=256, sr=16000, output_format="Magnitude"),
                      (1, 70000), {}),
}


def _forward(mod, x, reserve):
    """(mod(x), persistent-grid ledger of the call) under an SM reserve of ``reserve``."""
    old = _C.set_sm_reserve(reserve)
    _C.persistent_grid_read()
    try:
        with torch.no_grad(), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            y = mod(x)
        torch.cuda.synchronize()
    finally:
        _C.set_sm_reserve(old)
    return y, _C.persistent_grid_read()


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_full_grid_equals_single_cta_bitwise(name):
    cls, ctor, shape, kw = CONFIGS[name]
    mod = build(cls, ctor).cuda()
    xn = np.random.RandomState(5).standard_normal(shape).astype(np.float32)
    x = torch.from_numpy(xn).cuda()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    before = _C.launch_count()
    full, ledger_full = _forward(mod, x, 0)
    assert _C.launch_count() > before
    single, ledger = _forward(mod, x, sms - 1)
    # every persistent launch of the single-CTA leg ran one CTA; the full grid ran more
    n = ledger[0]
    assert n >= 1 and ledger == (n, n, 1, 1), (name, ledger)
    assert ledger_full[0] == n and ledger_full[3] > 1, (name, ledger_full)
    assert full.shape == single.shape
    # (the fused Mel epilogue adds at most two partial sums per filter: its atomic adds commute)
    assert torch.equal(full, single)
    emax, el2 = rel_errors(full.cpu().numpy(), run_oracle(cls, mod, xn, kw))
    assert emax < 1e-4 and el2 < 1e-4, (emax, el2)
