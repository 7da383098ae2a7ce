"""GPU: StreamingTransform / StreamingInverse against the offline module and the fp64 oracle.

On the tensor-core routes the concatenated pushes are bitwise ``module(x)`` (``_strict=True``: the fused chunk
route ran, no concat fallback) and within 1e-4 of the oracle; the concat route (``NNAUDIO_B200_PATH=simt``)
matches the offline SIMT output.  The streamed inverse is within 1e-6 of the offline inverse (both overlap-add
with fp32 atomics) and 1e-4 of the oracle.
"""
import numpy as np
import pytest
import torch

from helpers import rel_errors, run_oracle
from nnaudio_b200 import _C, features
from nnaudio_b200.streaming import StreamingInverse, StreamingTransform
from oracle import nnaudio_oracle as oracle

pytestmark = pytest.mark.gpu


def _chunkings(L, seed, n_random=3):
    rng = np.random.default_rng(seed)
    out = [[L]]
    for _ in range(n_random):
        cuts = np.sort(rng.integers(0, L + 1, size=rng.integers(1, 12)))
        out.append(list(np.diff(np.concatenate([[0], cuts, [L]]))))
    out.append([0, 1, 3, 0] + [L - 4])        # empty and tiny chunks at the start
    return out


def _stream(module, x, sizes, strict=True, **kw):
    st = StreamingTransform(module, x.shape[0], _strict=strict, **kw)
    parts, pos = [], 0
    for n in sizes:
        parts.append(st.push(x[:, pos:pos + int(n)]))
        pos += int(n)
    parts.append(st.flush())
    return torch.cat(parts, 2)


CASES = {
    # block-partial kernel, R = 4 and R = 2, every STFT format
    "stft_r4_mag": (lambda: features.STFT(n_fft=1024, hop_length=256, verbose=False), {}),
    "stft_r4_complex": (lambda: features.STFT(n_fft=1024, hop_length=256, output_format="Complex",
                                              verbose=False), {}),
    "stft_r4_phase": (lambda: features.STFT(n_fft=1024, hop_length=256, output_format="Phase", verbose=False), {}),
    "stft_r2_constant": (lambda: features.STFT(n_fft=512, hop_length=256, pad_mode="constant", verbose=False), {}),
    "stft_uncentred": (lambda: features.STFT(n_fft=1024, hop_length=256, center=False, verbose=False), {}),
    # dense kernel: non-Hann window, and a hop with several frame phases
    "stft_hamming": (lambda: features.STFT(n_fft=512, hop_length=128, window="hamming", verbose=False), {}),
    "stft_hop100": (lambda: features.STFT(n_fft=512, hop_length=100, verbose=False), {}),
    "mel_fused": (lambda: features.MelSpectrogram(sr=16000, n_fft=512, hop_length=128, n_mels=80,
                                                  verbose=False), {}),
    "gammatone": (lambda: features.Gammatonegram(sr=16000, n_fft=512, hop_length=128, n_bins=64,
                                                 verbose=False), {}),
    "mfcc": (lambda: features.MFCC(sr=16000, n_mfcc=20, n_fft=512, hop_length=128, top_db=None,
                                   verbose=False), {}),
    "cqt1992v2": (lambda: features.CQT1992v2(sr=16000, hop_length=128, fmin=55, n_bins=60, verbose=False), {}),
    "cqt1992v2_complex": (lambda: features.CQT1992v2(sr=16000, hop_length=128, fmin=55, n_bins=60,
                                                     output_format="Complex", verbose=False),
                          {"normalization_type": "wrap"}),
    "cqt1992": (lambda: features.CQT1992(sr=8000, hop_length=64, fmin=200, n_bins=24), {}),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_pushes_equal_offline_bitwise(name):
    make, kw = CASES[name]
    torch.manual_seed(0)
    m = make().cuda()
    x = torch.randn(3, 12000, device="cuda")
    with torch.no_grad():
        ref = m(x, **kw)
        for i, sizes in enumerate(_chunkings(x.shape[1], seed=len(name) * 31)):
            got = _stream(m, x, sizes, **kw)
            assert got.shape == ref.shape, (name, i)
            assert torch.equal(got, ref), (name, i, sizes, (got - ref).abs().max().item())
    want = run_oracle(type(m).__name__, m, x.cpu().numpy(), kw)
    got = got.cpu().numpy()
    if "phase" in name:  # an angle near pi (DC / Nyquist rows: imag 0 in fp64) lands on either side of the cut
        got = want + np.remainder(got - want + np.pi, 2 * np.pi) - np.pi
    emax, el2 = rel_errors(got, want)
    assert (el2 if "phase" in name else emax) <= 1e-4, (name, emax, el2)


def test_single_sample_pushes():
    m = features.MelSpectrogram(sr=16000, n_fft=512, hop_length=128, n_mels=80, verbose=False).cuda()
    x = torch.randn(2, 700, device="cuda")
    with torch.no_grad():
        assert torch.equal(_stream(m, x, [1] * 700), m(x))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("name", ["stft_r4_mag", "mel_fused", "cqt1992v2"])
def test_16bit_chunks_equal_upcast_offline(name, dtype):
    make, kw = CASES[name]
    m = make().cuda()
    x = torch.randn(2, 9000, device="cuda").to(dtype)
    with torch.no_grad():
        ref = m(x.float(), **kw)
        assert torch.equal(_stream(m, x, [1000, 17, 4000, 3983], **kw), ref)


def test_concat_route_under_simt(monkeypatch):
    monkeypatch.setenv("NNAUDIO_B200_PATH", "simt")
    m = features.STFT(n_fft=512, hop_length=128, verbose=False).cuda()
    x = torch.randn(2, 5000, device="cuda")
    with torch.no_grad():
        ref = m(x)
        with pytest.raises(RuntimeError, match="no fused chunk route"):
            _stream(m, x, [2500, 2500], strict=True)
        got = _stream(m, x, [2500, 7, 2493], strict=False)
    assert got.shape == ref.shape
    assert (got - ref).abs().max().item() <= 1e-6 * ref.abs().max().item()


def test_full_size_mel_batch_equal_offline():
    """cfg2: 64 x 10 s at 22.05 kHz in 100 ms pushes."""
    m = features.MelSpectrogram(sr=22050, n_fft=2048, hop_length=512, n_mels=128, verbose=False).cuda()
    x = torch.randn(64, 220500, device="cuda")
    with torch.no_grad():
        ref = m(x)
        got = _stream(m, x, [2205] * 100)
    assert torch.equal(got, ref), (got - ref).abs().max().item()


def test_full_size_cqt_batch_equal_offline(monkeypatch):
    """cfg3: 128 x 10 s at 44.1 kHz in 0.5 s pushes.  The whole-clip call has enough tiles for the tall
    kernel's balanced schedule, which sums a shared tile's two halves in another order (2e-6 of the static
    schedule, tests/test_zz_gpu_tall_balance.py), and whether a launch takes it depends on its tile count.
    On one schedule the pushes are bitwise the whole-clip result; across the two they are within 2e-6."""
    m = features.CQT1992v2(sr=44100, n_bins=84, bins_per_octave=12, fmin=32.7, verbose=False).cuda()
    x = torch.randn(128, 441000, device="cuda")
    with torch.no_grad():
        ref_default = m(x)
        got_default = _stream(m, x, [22050] * 20)
        monkeypatch.setenv("NNAB_TALL_BALANCE", "0")
        ref_static = m(x)
        got_static = _stream(m, x, [22050] * 20)
    assert torch.equal(got_static, ref_static), (got_static - ref_static).abs().max().item()
    assert (got_default - ref_default).abs().max().item() <= 2e-6 * ref_default.abs().max().item()


def test_push_does_not_synchronise():
    m = features.MelSpectrogram(sr=16000, n_fft=512, hop_length=128, n_mels=80, verbose=False).cuda()
    x = torch.randn(256, 3200, device="cuda")
    st = StreamingTransform(m, 256, _strict=True)
    with torch.no_grad():
        st.push(x[:, :320])  # first push: any lazy init happens outside the checked window
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for i in range(1, 10):
                st.push(x[:, 320 * i:320 * (i + 1)])
        finally:
            torch.cuda.set_sync_debug_mode(0)


# ---------------------------------------------------------------------------------------------------- inverse
def _istream(st, X, sizes, length=None):
    parts, pos = [], 0
    for t in sizes:
        parts.append(st.push(X[:, :, pos:pos + t]))
        pos += t
    assert pos == X.shape[2]
    parts.append(st.flush(length))
    return torch.cat(parts, 1)


@pytest.mark.parametrize("onesided", [True, False])
@pytest.mark.parametrize("kind", ["stft_inverse", "istft"])
def test_streamed_inverse_matches_offline_and_oracle(kind, onesided):
    torch.manual_seed(3)
    if kind == "stft_inverse":
        m = features.STFT(n_fft=1024, hop_length=256, iSTFT=True, verbose=False).cuda()
        kc, ks = m.kernel_cos_inv, m.kernel_sin_inv
    else:
        m = features.iSTFT(n_fft=512, hop_length=128, verbose=False).cuda()
        kc, ks = m.kernel_cos, m.kernel_sin
    n_fft = m.n_fft
    f_in = n_fft // 2 + 1 if onesided else n_fft
    X = torch.randn(3, f_in, 150, 2, device="cuda")
    with torch.no_grad():
        for length in (None, 150 * m.stride - 7):
            ref = m.inverse(X, onesided=onesided, length=length) if kind == "stft_inverse" else \
                m(X, onesided=onesided, length=length)
            st = StreamingInverse(m, 3, onesided=onesided)
            for sizes in ([150], [1] * 150, [0, 3, 0, 40, 7, 100]):
                st.reset()
                got = _istream(st, X, sizes, length)
                assert got.shape == ref.shape, (sizes, got.shape, ref.shape)
                peak = ref.abs().max().item()
                assert (got - ref).abs().max().item() <= 1e-6 * peak, (sizes, length)
            want = oracle.istft(X.cpu().numpy(), kc.cpu().numpy(), ks.cpu().numpy(), m.window_mask.cpu().numpy(),
                                m.stride, center=m.center, onesided=onesided, length=length)
            emax, _ = rel_errors(got.cpu().numpy(), want)
            assert emax <= 1e-4, (length, emax)


@pytest.mark.parametrize("n_fft,hop", [(512, 128), (1024, 256), (2048, 512)])
def test_reference_round_trip_with_streamed_inverse(n_fft, hop):
    """The reference's STFT -> inverse round trip (Installation/tests/test_stft.py, test_inverse), with the
    inverse streamed in blocks of frames."""
    stft = features.STFT(n_fft=n_fft, hop_length=hop, window="hann", iSTFT=True, verbose=False).cuda()
    x = torch.randn(4, 16000, device="cuda")
    with torch.no_grad():
        X = stft(x, output_format="Complex")
        st = StreamingInverse(stft, 4)
        T = X.shape[2]
        recon = _istream(st, X, [5, 0, 1] + [10] * ((T - 6) // 10) + [(T - 6) % 10], length=x.shape[1])
    assert np.allclose(x.cpu(), recon.cpu(), rtol=1e-5, atol=1e-3)


def test_streamed_inverse_push_does_not_synchronise():
    m = features.iSTFT(n_fft=512, hop_length=128, verbose=False).cuda()
    X = torch.randn(64, 257, 40, 2, device="cuda")
    st = StreamingInverse(m, 64, onesided=True)
    with torch.no_grad():
        st.push(X[:, :, :4])
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for i in range(1, 10):
                st.push(X[:, :, 4 * i:4 * (i + 1)])
        finally:
            torch.cuda.set_sync_debug_mode(0)
