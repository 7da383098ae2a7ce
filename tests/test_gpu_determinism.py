"""Run-to-run repeatability of the CUDA path (-m gpu): the reference is deterministic, so every
forward transform must return bit-identical results when called twice (VERDICT r1 item 5).
Split-K partial sums are combined by ordered read-modify-writes of one thread, the fused filterbank
gets at most two partial sums per filter (commutative), nothing else accumulates through atomics.
The dense kernel fuses a bank only when its tile cut allows that bound (else the un-fused GEMM runs).
The block-partial kernel's fused Mel keeps it at power 2 with a width the table builder found; a bank
with no such width, or power != 2, is outside this claim (test_zz_gpu_block_domain.py)."""
import numpy as np
import pytest
import torch

from helpers import build

pytestmark = pytest.mark.gpu

CASES = [
    ("STFT", dict(n_fft=2048, hop_length=512, output_format="Magnitude"), (6, 60000), {}),
    ("STFT", dict(n_fft=512, hop_length=160, output_format="Complex"), (3, 16000), {}),
    ("MelSpectrogram", dict(sr=22050, n_fft=2048, hop_length=512, n_mels=128), (8, 110250), {}),
    ("MelSpectrogram", dict(sr=16000, n_fft=1024, hop_length=256, n_mels=80), (5, 48000), {}),
    ("MelSpectrogram", dict(sr=22050, n_fft=2048, hop_length=300, n_mels=128), (3, 50000), {}),
    ("MFCC", dict(sr=16000), (8, 80000), {}),
    ("Gammatonegram", dict(sr=22050, n_fft=2048, hop_length=512), (4, 66150), {}),
    ("CQT1992v2", dict(sr=44100, n_bins=84, fmin=32.7), (4, 220500), {}),
    ("CQT1992v2", dict(sr=22050, n_bins=60, fmin=110.0), (3, 44100), dict(output_format="Complex")),
    ("CQT2010v2", dict(sr=22050, n_bins=88), (4, 132300), {}),
    ("VQT", dict(sr=22050, gamma=5), (2, 66150), {}),
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}-{i}" for i, c in enumerate(CASES)])
def test_forward_is_bit_repeatable(case):
    cls, ctor, shape, kw = case
    mod = build(cls, ctor).cuda()
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(7)).cuda()
    outs = []
    with torch.no_grad():
        for rep in range(4):
            # perturb allocator / cache state and the SMs' tile order between repetitions
            junk = torch.randn(1 << (18 + rep), device="cuda")
            outs.append(mod(x, **kw).clone())
            del junk
    torch.cuda.synchronize()
    for o in outs[1:]:
        assert torch.equal(outs[0], o), (cls, float((outs[0] - o).abs().max()))
