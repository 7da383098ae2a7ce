"""Balanced ("stream-K") schedule of the tall-A CQT kernel (-m gpu): the (tile, column chunk) units are cut
into equal ranges per CTA, a tile shared by two CTAs is finished through scratch + flags
(csrc/tct_kernels.cu: TallSched<true>).  NNAB_TALL_BALANCE=1 selects it, NNAB_TALL_CTAS shrinks the grid so
that small problems have shared tiles.  Checks: the balanced launch really ran (library counter), results
equal the static schedule up to the re-association of the fp32 chunk sums, stay within 1e-4 of the CPU
oracle, and are bit-identical run to run."""
import os
import warnings

import numpy as np
import pytest
import torch

from helpers import build, rel_errors, run_oracle

pytestmark = pytest.mark.gpu


def _forward(mod, x, balance, ctas=None, **kw):
    os.environ["NNAB_TALL_BALANCE"] = "1" if balance else "0"
    if ctas is not None:
        os.environ["NNAB_TALL_CTAS"] = str(ctas)
    try:
        with torch.no_grad(), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            y = mod(x, **kw)
        torch.cuda.synchronize()
    finally:
        os.environ.pop("NNAB_TALL_BALANCE", None)
        os.environ.pop("NNAB_TALL_CTAS", None)
    return y


@pytest.mark.parametrize("fmt", ["Magnitude", "Complex"])
@pytest.mark.parametrize("ctas", [4, 7])
def test_shared_tiles_match_static_schedule_and_oracle(ctas, fmt):
    from nnaudio_b200 import _C

    # K = 16384, hop 512: 8 column chunks; 48 clips x 76 frame slots = 29 tiles of 128 frames, shared by
    # 4 / 7 CTAs (the split-K scratch of the problem, 2 * 48 * 84 * 44 floats, holds 7 slots of 96 KB)
    mod = build("CQT1992v2", dict(sr=22050, n_bins=84)).cuda()
    x = torch.from_numpy(np.random.RandomState(7).standard_normal((48, 22050)).astype(np.float32)).cuda()
    kw = dict(output_format=fmt)
    static = _forward(mod, x, False, ctas, **kw)
    before = _C.balanced_launch_count()
    a = _forward(mod, x, True, ctas, **kw)
    assert _C.balanced_launch_count() == before + 1, "the balanced schedule was not selected"
    b = _forward(mod, x, True, ctas, **kw)
    assert torch.equal(a, b), "shared tiles must be summed in a fixed order"
    emax, el2 = rel_errors(a.cpu().numpy(), static.cpu().numpy())
    assert emax < 2e-6 and el2 < 2e-6, (emax, el2)
    for clip in (0, 47):
        ref = run_oracle("CQT1992v2", mod, x[clip:clip + 1].cpu().numpy(), kw)
        emax, el2 = rel_errors(a[clip:clip + 1].cpu().numpy(), ref)
        assert emax < 1e-4 and el2 < 1e-4, (clip, emax, el2)


def test_cfg3_full_size_balanced_equals_static():
    """BASELINE cfg3 (128 x 10 s @ 44.1 kHz): over 900 tiles of 128 frames on the full grid."""
    from nnaudio_b200 import _C

    mod = build("CQT1992v2", dict(sr=44100, n_bins=84, bins_per_octave=12, fmin=32.7)).cuda()
    g = torch.Generator(device="cuda").manual_seed(99)
    x = torch.randn(128, 441000, generator=g, device="cuda", dtype=torch.float32)
    static = _forward(mod, x, False)
    before = _C.balanced_launch_count()
    a = _forward(mod, x, True)
    assert _C.balanced_launch_count() == before + 1
    b = _forward(mod, x, True)
    assert torch.equal(a, b)
    d = (a - static).abs().max().item() / static.abs().max().item()
    assert d < 2e-6, d
