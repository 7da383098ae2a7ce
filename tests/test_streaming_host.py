"""CPU: the host logic of nnaudio_b200.streaming against whole-clip float64 stand-ins for the C calls.

Forward: two stand-ins for the ``_C.*_chunk_forward`` calls: "fused" returns the frames the library must return (the
float64 transform of the stream received so far, frames [frames, frames + T)); "concat" reports
NNAB_EUNSUPPORTED, so the streamer's own concat route (virtual clip, padding, carry ring) runs on the offline
stand-in.  Either way the concatenated pushes must equal the whole clip, and every push must return exactly
the frames whose samples have all arrived.  The CUDA kernels behind the fused route are checked on the GPU
(tests/test_zz_gpu_streaming.py).  Inverse: a stand-in that returns the requested samples of the offline inverse
of the frames received so far; the concatenation must equal the offline inverse of all frames.
"""
import ctypes

import numpy as np
import pytest
import torch

import cpu_kernels
from nnaudio_b200 import _C, features
from nnaudio_b200.streaming import StreamingInverse, StreamingTransform


# float64 end to end (cpu_kernels rounds its outputs to float32): the whole-clip reference and the streamed
# frames then agree to float64 round-off
def _format64(c, out_format, sqrt_eps):
    re, im = c[..., 0], c[..., 1]
    if out_format == _C.FMT_COMPLEX:
        return c
    if out_format == _C.FMT_MAGNITUDE:
        return torch.sqrt(re * re + im * im + sqrt_eps)
    if out_format == _C.FMT_PHASE_ANGLE:
        return torch.atan2(im, re)
    ang = torch.atan2(im, re)
    return torch.stack((torch.cos(ang), torch.sin(ang)), -1)


def stft_forward(x, wcos, wsin, packed, n_fft, hop, center, pad_mode, out_format, sqrt_eps, path=None):
    c = cpu_kernels._framed(x, cpu_kernels._mat(wcos), cpu_kernels._mat(wsin), hop, center, pad_mode)
    return _format64(c, out_format, sqrt_eps)


def stft_filterbank_forward(x, wcos, wsin, packed, n_fft, hop, center, pad_mode, sqrt_eps, power, fb,
                            fb_table=None, path=None):
    return cpu_kernels._mel_power(x, wcos, wsin, hop, center, pad_mode, sqrt_eps, power, fb)


def mfcc_forward(x, wcos, wsin, packed, n_fft, hop, center, pad_mode, sqrt_eps, power, mel_basis, amin, ref,
                 top_db, dct, fb_table=None, path=None):
    assert top_db is None
    S = cpu_kernels._mel_power(x, wcos, wsin, hop, center, pad_mode, sqrt_eps, power, mel_basis)
    db = 10.0 * torch.log10(torch.clamp(S, min=amin)) - 10.0 * np.log10(max(amin, abs(ref)))
    return torch.matmul(dct.double(), db)


def cqt1992v2_forward(x, k_real, k_imag, packed, k_begin, k_end, hop, center, pad_mode, scale, scale_all,
                      out_format, sqrt_eps, path=None):
    c = cpu_kernels._framed(x, k_real, k_imag, hop, center, pad_mode)
    return _format64(cpu_kernels._scaled(c, scale, scale_all), out_format, sqrt_eps)


_OFFLINE64 = {"stft_forward": stft_forward, "stft_filterbank_forward": stft_filterbank_forward,
              "mfcc_forward": mfcc_forward, "cqt1992v2_forward": cqt1992v2_forward}


def _fused_standin(name):
    offline = _OFFLINE64[name]
    shadow = {}

    def chunk_forward(st, x, flush, T, **kw):
        buf = shadow.setdefault(id(st), [])
        if st.received == 0:
            buf.clear()
        if x is not None and x.shape[-1] > 0:
            buf.append(x.float())
        if T == 0:
            return st._empty(name, kw)
        whole = torch.cat(buf, 1)
        full = offline(whole, **kw)
        assert full.shape[2] >= st.frames + T
        return full[:, :, st.frames:st.frames + T]

    return chunk_forward


def _install(monkeypatch, mode):
    cpu_kernels.install(monkeypatch)
    for name in _OFFLINE64:
        monkeypatch.setattr(_C, name, _OFFLINE64[name])
        fn = _fused_standin(name) if mode == "fused" else (lambda *a, **k: None)
        monkeypatch.setattr(_C, name.replace("_forward", "_chunk_forward"), fn)


def _needed_frames(total, K, hop, center, reflect):
    """Brute force: frames every raw sample of which has arrived, by listing the samples each frame reads."""
    pad = K // 2 if center else 0
    t = 0
    while True:
        idx = np.arange(t * hop - pad, t * hop - pad + K)
        if reflect:
            idx = np.where(idx < 0, -idx, idx)
        if idx.max() >= total:
            return t
        t += 1


CONFIGS = {
    "stft_mag": (lambda: features.STFT(n_fft=64, hop_length=16, verbose=False), {}),
    "stft_complex": (lambda: features.STFT(n_fft=64, hop_length=16, output_format="Complex", verbose=False), {}),
    "stft_phase": (lambda: features.STFT(n_fft=64, hop_length=16, output_format="Phase", verbose=False), {}),
    "stft_constant": (lambda: features.STFT(n_fft=64, hop_length=16, pad_mode="constant", verbose=False), {}),
    "stft_uncentred": (lambda: features.STFT(n_fft=64, hop_length=16, center=False, verbose=False), {}),
    "stft_r2": (lambda: features.STFT(n_fft=64, hop_length=32, verbose=False), {}),
    "stft_hop_half_reflect": (lambda: features.STFT(n_fft=48, hop_length=24, verbose=False), {}),
    "stft_hamming_hop12": (lambda: features.STFT(n_fft=64, hop_length=12, window="hamming", verbose=False), {}),
    "mel": (lambda: features.MelSpectrogram(sr=8000, n_fft=64, hop_length=16, n_mels=12, verbose=False), {}),
    "gammatone": (lambda: features.Gammatonegram(sr=8000, n_fft=64, hop_length=16, n_bins=12, verbose=False), {}),
    "mfcc": (lambda: features.MFCC(sr=8000, n_mfcc=8, n_fft=64, hop_length=16, n_mels=12, top_db=None,
                                   verbose=False), {}),
    "cqt1992v2": (lambda: features.CQT1992v2(sr=8000, hop_length=64, fmin=400, n_bins=24, verbose=False), {}),
    "cqt1992v2_complex_wrap": (lambda: features.CQT1992v2(sr=8000, hop_length=64, fmin=400, n_bins=24,
                                                          output_format="Complex", verbose=False),
                               {"normalization_type": "wrap"}),
    "cqt1992": (lambda: features.CQT1992(sr=8000, hop_length=64, fmin=400, n_bins=12), {}),
}


def _chunkings(L, K, hop, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(5):
        cuts = np.sort(rng.integers(0, L + 1, size=rng.integers(1, 10)))
        out.append([int(v) for v in np.diff(np.concatenate([[0], cuts, [L]]))])
    out.append([L])                                       # one chunk holding everything
    out.append([1] * 40 + [L - 40])                       # 1-sample chunks
    out.append([0, 0, hop - 1, 0, K // 2 - 1, 1, 1] + [L - hop - K // 2])  # empty, < hop, < n_fft // 2
    return out


@pytest.mark.parametrize("mode", ["fused", "concat"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_concatenated_pushes_equal_whole_clip(name, mode, monkeypatch):
    _install(monkeypatch, mode)
    make, kw = CONFIGS[name]
    m = make()
    L = 1500
    torch.manual_seed(1)
    x = torch.randn(2, L)
    ref = m(x, **kw)
    st = StreamingTransform(m, 2, **kw)
    for sizes in _chunkings(L, st.K, st.hop, seed=len(name)):
        st.reset()
        parts, pos = [], 0
        for n in sizes:
            out = st.push(x[:, pos:pos + n])
            pos += n
            parts.append(out)
            assert st.frames == _needed_frames(pos, st.K, st.hop, st.pad > 0, st._reflect), (name, sizes)
        assert pos == L
        parts.append(st.flush())
        got = torch.cat(parts, 2)
        assert got.shape == ref.shape, (name, sizes)
        d = got - ref
        if name == "stft_phase":  # float64 round-off may put an angle of pi on either side of the cut
            d = torch.remainder(d + np.pi, 2 * np.pi) - np.pi
        assert d.abs().max().item() <= 1e-12 * ref.abs().max().item(), (name, mode, sizes)


def test_mfcc_top_db_and_unsupported_modules_rejected():
    with pytest.raises(ValueError, match="top_db"):
        StreamingTransform(features.MFCC(sr=8000, n_fft=64, hop_length=16, n_mels=12, verbose=False), 1)
    for m in (features.CQT2010v2(sr=8000, n_bins=12, fmin=400, verbose=False),
              features.VQT(sr=8000, n_bins=12, fmin=400, verbose=False),
              features.CQT2010(sr=8000, n_bins=12, fmin=400, verbose=False),
              features.CFP(fs=8000), features.Combined_Frequency_Periodicity(fr=2, fs=8000),
              features.Griffin_Lim(n_fft=64, hop_length=16),
              features.iSTFT(n_fft=64, hop_length=16, verbose=False)):
        with pytest.raises(TypeError):
            StreamingTransform(m, 1)


def test_rules(monkeypatch):
    _install(monkeypatch, "fused")
    m = features.STFT(n_fft=64, hop_length=16, verbose=False)
    with pytest.raises(ValueError):
        StreamingTransform(m, 65536)
    st = StreamingTransform(m, 2)
    st.push(torch.zeros(2, 10))
    with pytest.raises(ValueError):
        st.push(torch.zeros(2, 10, dtype=torch.bfloat16))  # dtype fixed at the first push
    with pytest.raises(ValueError):
        st.push(torch.zeros(3, 10))  # batch fixed
    with pytest.raises(NotImplementedError):
        st.push(torch.zeros(2, 10, requires_grad=True))
    # a stream too short for the module: the exception type module(x) raises (AssertionError: L < pad)
    with pytest.raises(AssertionError):
        st.flush()
    st.reset()
    st.push(torch.zeros(2, 32))
    with pytest.raises(RuntimeError):
        st.flush()  # L == pad: reflect padding needs pad < L
    st.reset()
    st.push(torch.randn(2, 100))
    st.flush()
    with pytest.raises(RuntimeError):
        st.push(torch.zeros(2, 1))
    st.reset()
    assert st.push(torch.randn(2, 100)).shape[2] == _needed_frames(100, 64, 16, True, True)


def test_chunk_entry_points_reject_bad_arguments_on_the_host():
    lib = _C.lib()
    P = ctypes.c_void_p
    ring = chunk = w = out = P(256)  # never dereferenced on the host
    EINVAL = -1

    def stft(received=0, n_carry=0, frames=0, n=100, T=3, flush=0, dtype=0, B=2, st=ring, pitch=100):
        return lib.nnab_stft_chunk_forward(st, received, n_carry, frames, chunk, dtype, B, n, pitch, flush, w, w,
                                           None, 64, 33, 16, 1, 0, 0, 0.0, out, T, None, 0, 0, None)

    # after 100 samples (n_fft 64, hop 16, reflect): frames t with 16 t + 32 <= 100 -> 5
    assert stft(T=4) == EINVAL, "T must be the frames this push completes"
    assert stft(st=None) == EINVAL
    assert stft(dtype=9) == EINVAL
    assert stft(B=65536) == EINVAL
    assert stft(pitch=50) == EINVAL
    assert stft(received=100, n_carry=10, frames=5, n=0, T=0) == EINVAL, "counters no stream can have"
    assert stft(received=100, n_carry=36, frames=4, n=0, T=0) == EINVAL, "frames must be every ready frame"
    assert stft(received=20, n_carry=20, frames=0, n=0, T=0, flush=1) == EINVAL, "reflect needs pad < L"
    assert lib.nnab_mfcc_chunk_forward(ring, 0, 0, 0, chunk, 0, 2, 100, 100, 0, w, w, None, 64, 33, 16, 1, 0,
                                       0.0, 2.0, w, 12, None, 1e-10, 1.0, 80.0, w, 8, out, 5, None, 0, 0,
                                       None) == EINVAL, "top_db is a whole-clip maximum"
    # host-only size queries
    assert lib.nnab_chunk_state_bytes(3, 64) == 3 * 64 * 4
    assert lib.nnab_stft_chunk_workspace_bytes(2, 0, 0, 10, 0, 64, 33, 16, 1, 0, _C.PATH_SIMT) == 0
    assert lib.nnab_stft_chunk_workspace_bytes(2, 0, 0, 100, 0, 64, 33, 16, 1, 0, _C.PATH_AUTO) == \
        lib.nnab_stft_workspace_bytes(2, 16 * 4 + 64, 64, 33, 16, 0, _C.PATH_AUTO)


# ---------------------------------------------------------------------------------------------------- inverse
def _install_inverse(monkeypatch):
    cpu_kernels.install(monkeypatch)
    shadow = {}

    def istft_chunk_forward(st, X, flush, length, n_out, packed, window, n_fft, hop, center):
        frames = shadow.setdefault(id(st), [])
        if st.frames == 0:
            frames.clear()
        frames.append(X)
        allX = torch.cat(frames, 2)
        # positions below frames * hop are final: the offline inverse of the frames so far has them
        y = cpu_kernels.istft_forward(allX, packed, window, n_fft, hop, center, length if flush else None)
        out = y[:, st.emitted:st.emitted + n_out]
        assert out.shape[1] == n_out, (out.shape, n_out)
        return out

    monkeypatch.setattr(_C, "istft_chunk_forward", istft_chunk_forward)


INVERSE = {
    "istft_twosided": (lambda: features.iSTFT(n_fft=64, hop_length=16, verbose=False), False),
    "istft_onesided": (lambda: features.iSTFT(n_fft=64, hop_length=16, verbose=False), True),
    "istft_uncentred_hop_half": (lambda: features.iSTFT(n_fft=64, hop_length=32, center=False, verbose=False),
                                 True),
    "stft_inverse": (lambda: features.STFT(n_fft=64, hop_length=16, iSTFT=True, verbose=False), True),
    "istft_hop_gt_half": (lambda: features.iSTFT(n_fft=64, hop_length=40, verbose=False), True),
}


@pytest.mark.parametrize("length", [None, 1590, 5000])  # None, within the overlap-add span, past its end
@pytest.mark.parametrize("name", sorted(INVERSE))
def test_streamed_inverse_equals_offline(name, length, monkeypatch):
    _install_inverse(monkeypatch)
    make, onesided = INVERSE[name]
    m = make()
    f_in = 33 if onesided else 64
    torch.manual_seed(2)
    X = torch.randn(2, f_in, 40, 2)
    if isinstance(m, features.STFT):
        ref = m.inverse(X, onesided=onesided, length=length)
    else:
        ref = m(X, onesided=onesided, length=length)
    st = StreamingInverse(m, 2, onesided=onesided)
    for sizes in ([40], [1] * 40, [0, 1, 0, 7, 13, 19], [3, 0, 37]):
        st.reset()
        parts, pos = [], 0
        for t in sizes:
            parts.append(st.push(X[:, :, pos:pos + t]))
            pos += t
        parts.append(st.flush(length))
        got = torch.cat(parts, 1)
        assert got.shape == ref.shape, (name, sizes, got.shape, ref.shape)
        assert (got - ref).abs().max().item() <= 1e-6 * ref.abs().max().item(), (name, sizes)


def test_inverse_rules(monkeypatch):
    _install_inverse(monkeypatch)
    m = features.iSTFT(n_fft=64, hop_length=16, verbose=False)
    with pytest.raises(TypeError):
        StreamingInverse(features.STFT(n_fft=64, hop_length=16, verbose=False), 1)  # no iSTFT=True
    with pytest.raises(ValueError):
        StreamingInverse(m, 65536)
    st = StreamingInverse(m, 2, onesided=True)
    with pytest.raises(RuntimeError):
        st.flush()  # no frame yet
    with pytest.raises(ValueError):
        st.push(torch.zeros(2, 64, 3, 2))  # bins of a two-sided spectrum
    with pytest.raises(NotImplementedError):
        st.push(torch.zeros(2, 33, 3, 2, requires_grad=True))
    st.push(torch.randn(2, 33, 20, 2))
    with pytest.raises(ValueError):
        st.flush(length=10)  # shorter than what was already returned
    st.flush()
    with pytest.raises(RuntimeError):
        st.push(torch.zeros(2, 33, 1, 2))


def test_istft_chunk_entry_point_rejects_bad_counters_and_sizes_a_pool_workspace():
    lib = _C.lib()
    P = ctypes.c_void_p
    p = P(256)
    EINVAL = -1

    def call(frames=0, emitted=0, T=4, flush=0, length=-1, out_len=None, hop=16, center=1):
        if out_len is None:  # 4 frames, n_fft 64, hop 16, centred: positions [32, 64) are final
            out_len = 32
        return lib.nnab_istft_chunk_forward(p, frames, emitted, p, 2, 33, T, p, p, 64, hop, center, flush, length,
                                            p, out_len, None, 0, None)

    assert call(out_len=31) == EINVAL, "out_len must be the samples this push completes"
    assert call(frames=4, emitted=3, T=0, out_len=0) == EINVAL, "counters no stream has"
    assert call(frames=4, emitted=32, T=0, flush=1, length=10, out_len=0) == EINVAL, "length < returned"
    assert call(hop=65) == EINVAL, "frames that do not overlap"
    assert call(frames=0, T=0, flush=1, out_len=0) == EINVAL, "flush without frames"
    # the push is the pool push of its B lanes: the pool layout, a lead of n_fft positions per overlap-add row
    assert lib.nnab_istft_chunk_workspace_bytes(2, 33, 4, 64, 16) == \
        lib.nnab_istft_pool_workspace_bytes(2, 33, 4, 64, 16)
