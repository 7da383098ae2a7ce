"""GPU: StreamingPyramid against the offline CQT2010v2 / VQT / CQT2010 call and the fp64 oracle.

The pushes plus the flush, concatenated along time, are bitwise ``module(x)`` (16-bit chunks: bitwise
``module(x.float())``) on every all-tensor-core pyramid plan (generation 2: 256-wide FIR sources without early
downsampling; generation 1: early downsampling or other bank widths), and within 1e-4 of the oracle.
"""
import numpy as np
import pytest
import torch

from helpers import rel_errors, run_oracle
from nnaudio_b200 import features
from nnaudio_b200.streaming import StreamingPyramid

pytestmark = pytest.mark.gpu


def _chunkings(L, seed, n_random=3):
    rng = np.random.default_rng(seed)
    out = [[L]]
    for _ in range(n_random):
        cuts = np.sort(rng.integers(0, L + 1, size=rng.integers(1, 12)))
        out.append(list(np.diff(np.concatenate([[0], cuts, [L]]))))
    out.append([0, 1, 3, 0] + [1] * 300 + [0] + [L - 304])  # empty and 1-sample chunks
    return out


def _stream(module, x, sizes, **kw):
    st = StreamingPyramid(module, x.shape[0], **kw)
    parts, pos = [], 0
    for n in sizes:
        parts.append(st.push(x[:, pos:pos + int(n)]))
        pos += int(n)
    parts.append(st.flush())
    return torch.cat(parts, 2)


def _vqt(**kw):
    return lambda: features.VQT(sr=22050, n_bins=84, gamma=5, earlydownsample=False, verbose=False,
                                **{"hop_length": 512, **kw})


def _v2(**kw):
    return lambda: features.CQT2010v2(verbose=False, **{"sr": 22050, "hop_length": 512, "n_bins": 88, **kw})


CASES = {
    # generation 2 (22.05 kHz defaults: 256-wide banks, no early downsampling), every format, constant padding
    "v2_gen2": ("CQT2010v2", _v2(), {}),
    "v2_gen2_complex": ("CQT2010v2", _v2(n_bins=60, fmin=55), {"output_format": "Complex",
                                                                "normalization_type": "wrap"}),
    "v2_gen2_phase": ("CQT2010v2", _v2(n_bins=60, fmin=55), {"output_format": "Phase"}),
    "v2_constant": ("CQT2010v2", _v2(n_bins=60, fmin=55, pad_mode="constant"), {}),
    "v2_hop128": ("CQT2010v2", _v2(hop_length=128, n_bins=84), {}),  # low octaves with several frame phases
    "vqt_gamma0": ("VQT", lambda: features.VQT(sr=22050, hop_length=512, n_bins=84, gamma=0, verbose=False), {}),
    # generation 1 with early downsampling (44.1 kHz defaults), and CQT2010
    "v2_early": ("CQT2010v2", _v2(sr=44100, n_bins=84), {}),
    "cqt2010": ("CQT2010", lambda: features.CQT2010(sr=22050, hop_length=512, n_bins=84, verbose=False), {}),
    # VQT(gamma=5): bank widths 256 -> 64 across the octaves, so generation 1 without early downsampling
    "vqt_gamma5": ("VQT", _vqt(), {}),
    "vqt_complex": ("VQT", _vqt(), {"output_format": "Complex", "normalization_type": "wrap"}),
    "vqt_phase": ("VQT", _vqt(), {"output_format": "Phase"}),
    "vqt_constant": ("VQT", _vqt(pad_mode="constant"), {"normalization_type": "convolutional"}),
    # low octaves with several frame phases (hop_i < 8)
    "vqt_hop128": ("VQT", _vqt(hop_length=128), {}),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_pushes_equal_offline_and_oracle(name):
    cls, make, kw = CASES[name]
    m = make().cuda()
    L = 22050 * 2 + 333
    torch.manual_seed(3)
    x = torch.randn(3, L, device="cuda")
    ref = m(x, **kw)
    for sizes in _chunkings(L, seed=len(name)):
        y = _stream(m, x, sizes, **kw)
        assert y.shape == ref.shape, (name, sizes, y.shape, ref.shape)
        assert torch.equal(y, ref), (name, sizes, (y - ref).abs().max().item())
    want = run_oracle(cls, m, x.cpu().numpy(), kw)
    got = ref.cpu().numpy()
    if kw.get("output_format") == "Phase":
        # unit vectors: the phase of a bin with vanishing magnitude is ill-conditioned, compare the others
        c = run_oracle(cls, m, x.cpu().numpy(), dict(kw, output_format="Complex"))
        mag = np.hypot(c[..., 0], c[..., 1])
        keep = mag > 1e-2 * mag.max()
        assert np.abs(got - want)[keep].max() < 1e-3
    else:
        assert rel_errors(got, want)[0] < 1e-4, name


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("name", ["v2_gen2", "v2_early", "vqt_gamma5", "vqt_hop128"])
def test_half_chunks_equal_upcast(name, dtype):
    cls, make, kw = CASES[name]
    m = make().cuda()
    torch.manual_seed(4)
    x = torch.randn(2, 30000, device="cuda").to(dtype)
    ref = m(x.float(), **kw)
    for sizes in ([30000], [4097, 0, 1, 12000, 13902]):
        assert torch.equal(_stream(m, x, sizes, **kw), ref)


def test_full_size_cfg4():
    """cfg4: CQT2010v2, 256 streams x 30 s at 22.05 kHz, 88 bins, in 0.5 s pushes."""
    m = _v2()().cuda()
    L = 22050 * 30
    torch.manual_seed(5)
    x = torch.randn(256, L, device="cuda")
    ref = m(x)
    step = 22050 // 2
    sizes = [step] * (L // step) + [L % step]
    assert torch.equal(_stream(m, x, sizes), ref)


def test_steady_pushes_do_not_synchronise():
    m = _v2()().cuda()
    st = StreamingPyramid(m, 4)
    x = torch.randn(4, 22050, device="cuda")
    for i in range(3):  # warm-up: packed operands
        st.push(x[:, i * 2205:(i + 1) * 2205])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(3, 9):
            st.push(x[:, i * 2205:(i + 1) * 2205])
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_simt_path_raises_and_keeps_state(monkeypatch):
    m = _vqt()().cuda()
    x = torch.randn(2, 40000, device="cuda")
    st = StreamingPyramid(m, 2)
    st.push(x[:, :20000])
    before = (st.received, st.n_carry, st.frames, st.ring.clone())
    monkeypatch.setenv("NNAUDIO_B200_PATH", "simt")
    with pytest.raises(RuntimeError, match="no streamed tensor-core"):
        st.push(x[:, 20000:])
    assert (st.received, st.n_carry, st.frames) == before[:3]
    assert torch.equal(st.ring, before[3])
    monkeypatch.setenv("NNAUDIO_B200_PATH", "auto")
    st.reset()
    parts = [st.push(x[:, :20000]), st.push(x[:, 20000:]), st.flush()]
    assert torch.equal(torch.cat(parts, 2), m(x))
