"""The block-partial STFT kernel's epilogue (csrc/tcb_kernels.cu, epilogue_tile_block: frame sum before the Hann
window, tools/block_epilogue_emulation.py) against float64 references (-m gpu), on noise and on the inputs where the
window's 3-tap cancels hardest: a pure tone and a tone with noise 100 dB below it.  Shapes: cfg2's MelSpectrogram
(the warp-specialised kernel with its action lists in shared memory), Magnitude / Complex STFT-2048, MFCC (dB
output), the Gammatonegram's operand planes, and an R = 2 STFT.  Each case prints max|d| / max|ref|."""
import numpy as np
import pytest
import torch

import block_domain as bd
from conftest import record_error
from helpers import build, rel_errors, run_oracle

pytestmark = pytest.mark.gpu

BAR = 1e-4  # max|d| / max|ref| and ||d||_2 / ||ref||_2, the bar of test_gpu_parity.py and the block-domain tests


def _signal(kind, B, L, sr):
    t = np.arange(L)
    rng = np.random.RandomState(L + len(kind))
    if kind == "noise":
        return rng.standard_normal((B, L)).astype(np.float32)
    f0 = 440.0 * (1 + np.arange(B))[:, None] * 1.013
    x = np.sin(2 * np.pi * f0 / sr * t[None, :])
    if kind == "tone-100dB":
        x = x + 1e-5 * rng.standard_normal((B, L))
    return x.astype(np.float32)


SIGNALS = ["tone", "tone-100dB", "noise"]


@pytest.mark.parametrize("signal", SIGNALS)
@pytest.mark.parametrize("n_fft,hop,fmt", [(2048, 512, "Magnitude"), (2048, 512, "Complex"),
                                           (2048, 1024, "Magnitude"), (2048, 1024, "Complex")])
def test_stft_epilogue_vs_float64(n_fft, hop, fmt, signal):
    B, L = 2, 22050 * 2
    xn = _signal(signal, B, L, 22050)
    mod = build("STFT", dict(n_fft=n_fft, hop_length=hop)).cuda()
    with torch.no_grad():
        y = mod(torch.from_numpy(xn).cuda(), output_format=fmt).cpu().numpy().astype(np.float64)
    X = bd.ref_stft(xn, n_fft, hop)
    got = y[..., 0] + 1j * y[..., 1] if fmt == "Complex" else y
    want = X if fmt == "Complex" else np.abs(X)
    emax = float(np.abs(got - want).max() / np.abs(want).max())
    el2 = float(np.linalg.norm(got - want) / np.linalg.norm(want))
    case = f"{n_fft}/{hop} {fmt} {signal}"
    print(f"{case}: max|d|/max|ref| {emax:.2e}  l2 {el2:.2e}")
    record_error("block_epilogue_stft", case, max_rel=emax, l2_rel=el2)
    assert emax <= BAR and el2 <= BAR, (case, emax, el2)


FEATURES = {
    "cfg2_mel": ("MelSpectrogram", dict(sr=22050, n_fft=2048, hop_length=512, n_mels=128), 22050),
    "mfcc": ("MFCC", dict(sr=16000), 16000),
    "gammatone": ("Gammatonegram", dict(sr=22050, n_fft=2048, hop_length=512, n_bins=64), 22050),
}


@pytest.mark.parametrize("signal", SIGNALS)
@pytest.mark.parametrize("name", sorted(FEATURES))
def test_feature_epilogue_vs_float64(name, signal):
    cls, ctor, sr = FEATURES[name]
    B, L = 3, sr * 3
    xn = _signal(signal, B, L, sr)
    mod = build(cls, ctor).cuda()
    with torch.no_grad():
        y = mod(torch.from_numpy(xn).cuda())
    torch.cuda.synchronize()
    emax, el2 = rel_errors(y.cpu().numpy(), run_oracle(cls, mod, xn, {}))
    case = f"{name} {signal}"
    print(f"{case}: max|d|/max|ref| {emax:.2e}  l2 {el2:.2e}")
    record_error("block_epilogue_feature", case, max_rel=emax, l2_rel=el2)
    assert emax < BAR and el2 < BAR, (case, emax, el2)
