"""Host logic of StreamingPyramid (no GPU): the ready rule against a brute-force dependency listing, the
concatenation against the whole clip on a float64 stand-in of the chunk call, the flush exceptions, the
stream rules, the latency figure and the library's push plan (counters, read-back origins, ring capacity)."""
import numpy as np
import pytest
import torch

import cpu_kernels
from nnaudio_b200 import _C, features
from nnaudio_b200.streaming import StreamingPyramid, StreamingTransform


def _vqt(**kw):
    return lambda: features.VQT(sr=22050, n_bins=36, fmin=110, gamma=5, earlydownsample=False, verbose=False,
                                **{"hop_length": 128, **kw})


CONFIGS = {
    "vqt_reflect": (_vqt(), {}),
    "vqt_constant": (_vqt(pad_mode="constant"), {}),
    "vqt_complex": (_vqt(), {"output_format": "Complex", "normalization_type": "wrap"}),
    "vqt_phase": (_vqt(), {"output_format": "Phase"}),
    "vqt_multiphase": (_vqt(hop_length=16), {}),  # octave 2 frames every 4 samples
    # 256-wide banks: the generation-2 plan, whose ready rule waits one sample more per stage
    "cqt2010v2_gen2": (lambda: features.CQT2010v2(sr=22050, n_bins=36, fmin=220, hop_length=128,
                                                  earlydownsample=False, verbose=False), {}),
}


def _octaves64(x, kw):
    """Per-octave float64 frames of the pyramid on the samples so far (cpu_kernels.cqt_pyramid_forward
    without the equal-frame-count stacking)."""
    cur, hop, outs = x.double(), kw["hop"], []
    for i, (kr, ki) in enumerate(zip(kw["banks_real"], kw["banks_imag"])):
        if i > 0:
            cur = cpu_kernels.fir_decimate(cur, kw["lowpass"], 2).double()
            hop //= 2
        mode = kw["pad_mode"]
        if mode == _C.PAD_REFLECT and kr.shape[1] // 2 >= cur.shape[-1]:
            mode = _C.PAD_CONSTANT
        outs.insert(0, cpu_kernels._framed(cur, kr, ki, hop, True, mode))
    return outs


def _install(monkeypatch):
    cpu_kernels.install(monkeypatch)
    shadow = {}

    def chunk_forward(st, x, flush, T, **kw):
        buf = shadow.setdefault(id(st), [])
        if st.received == 0:
            buf.clear()
        if x is not None and x.shape[-1] > 0:
            buf.append(x.float())
        whole = torch.cat(buf, 1) if buf else torch.zeros(st.batch, 0)
        if T > 0:
            outs = _octaves64(whole, kw)
            c = torch.cat([o[:, :, st.frames:st.frames + T] for o in outs], 1)[:, -kw["n_bins"]:]
            assert c.shape[2] == T
            return cpu_kernels._format(cpu_kernels._scaled(c, kw["scale"], kw["scale_all"]), kw["out_format"],
                                       kw["sqrt_eps"])
        shape = (st.batch, kw["n_bins"], 0) if kw["out_format"] == _C.FMT_MAGNITUDE else (st.batch, kw["n_bins"], 0, 2)
        return torch.zeros(shape)

    monkeypatch.setattr(_C, "cqt_pyramid_chunk_forward", chunk_forward)


def _chunkings(L, seed):
    rng = np.random.default_rng(seed)
    out = [[L]]
    for _ in range(3):
        cuts = np.sort(rng.integers(0, L + 1, size=rng.integers(1, 10)))
        out.append(list(np.diff(np.concatenate([[0], cuts, [L]]))))
    out.append([0, 1, 0, 1] + [97] * 20 + [L - 1942])
    return out


def _brute_ready(st, received):
    """Frames final in every octave, by listing for each frame the raw samples it depends on: the octave's
    level samples (reflect mirror at the start), each level sample n through its FIR taps 2 n - 127 .. 2 n + 128
    of the level above (zero padding below 0); on the generation-2 plan one sample more per stage (its edge fix
    recomputes the whole clip's last 64 outputs of a stage)."""
    extra = 1 if st.generation == 2 else 0

    def last_raw(m, level):
        for _ in range(level):
            m = 2 * m + 128 + extra
        return m

    t = 0
    while True:
        for i, w in enumerate(st.widths):
            hop, pad = st.hop >> i, w // 2
            idx = np.arange(t * hop - pad, t * hop - pad + w)
            if st._reflect:
                idx = np.abs(idx)
            if last_raw(int(idx.max()), i) >= received:
                return t
        t += 1


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_concatenated_pushes_equal_whole_clip(name, monkeypatch):
    _install(monkeypatch)
    make, kw = CONFIGS[name]
    m = make()
    L = 3000
    torch.manual_seed(1)
    x = torch.randn(2, L)
    ref = m(x, **kw)
    st = StreamingPyramid(m, 2, **kw)
    for sizes in _chunkings(L, seed=len(name)):
        st.reset()
        parts, pos = [], 0
        for n in sizes:
            out = st.push(x[:, pos:pos + n])
            pos += n
            assert out.shape[2] == _brute_ready(st, pos) - (st.frames - out.shape[2]), (sizes, pos)
            parts.append(out)
        parts.append(st.flush())
        y = torch.cat(parts, 2)
        assert y.shape == ref.shape
        assert torch.allclose(y, ref, rtol=1e-6, atol=1e-6), (name, sizes)


def test_ready_rule_matches_dependency_listing(monkeypatch):
    _install(monkeypatch)
    for make, _ in CONFIGS.values():
        st = StreamingPyramid(make(), 1)
        for received in list(range(0, 1200, 7)) + [5000, 5001, 5002, 5003]:
            assert st._ready(received) == _brute_ready(st, received), received


def test_flush_raises_like_module(monkeypatch):
    _install(monkeypatch)
    m = _vqt()()
    raised = 0
    for L in range(1, 600, 3):
        try:
            m(torch.randn(1, L))
            continue
        except RuntimeError as e:  # octave frame counts that differ, or a level too short
            want = type(e)
        raised += 1
        st = StreamingPyramid(m, 1)
        st.push(torch.randn(1, L))
        with pytest.raises(want):
            st.flush()
    assert raised > 0


def test_rules(monkeypatch):
    _install(monkeypatch)
    m = _vqt()()
    with pytest.raises(ValueError):
        StreamingPyramid(m, 65536)
    with pytest.raises(TypeError):
        StreamingPyramid(features.STFT(n_fft=64, hop_length=16, verbose=False), 1)
    st = StreamingPyramid(m, 2)
    st.push(torch.zeros(2, 10))
    with pytest.raises(ValueError):
        st.push(torch.zeros(2, 10, dtype=torch.bfloat16))  # dtype fixed at the first push
    with pytest.raises(ValueError):
        st.push(torch.zeros(3, 10))
    with pytest.raises(NotImplementedError):
        st.push(torch.zeros(2, 10, requires_grad=True))
    st.push(torch.zeros(2, 3000))
    st.flush()
    with pytest.raises(RuntimeError):
        st.push(torch.zeros(2, 10))
    st.reset()
    assert (st.received, st.n_carry, st.frames, st.dtype) == (0, 0, 0, None)
    st.push(torch.zeros(2, 10, dtype=torch.float16))


def test_plans_and_rejected_configurations(monkeypatch):
    _install(monkeypatch)
    assert StreamingPyramid(features.CQT2010v2(sr=22050, n_bins=84, hop_length=512, verbose=False), 1).generation == 2
    early = StreamingPyramid(features.CQT2010v2(sr=44100, n_bins=84, hop_length=512, verbose=False), 1)
    assert early.generation == 1 and early.early > 1
    assert StreamingPyramid(_vqt()(), 1).generation == 1
    with pytest.raises(ValueError, match="multiple"):
        StreamingPyramid(_vqt(hop_length=102)(), 1)
    with pytest.raises(TypeError, match="StreamingPyramid"):
        StreamingTransform(_vqt()(), 1)


LATENCY_CFG4 = 32640


def test_latency_of_an_88_bin_stream(monkeypatch):
    """cfg4: CQT2010v2, 88 bins at 22.05 kHz, hop 512 (generation 2, 8 octaves): frame t returns once
    t * 512 + 32640 samples (1.48 s) have arrived.  Arithmetic of the ready rule, not a measurement."""
    _install(monkeypatch)
    st = StreamingPyramid(features.CQT2010v2(sr=22050, hop_length=512, n_bins=88, verbose=False), 1)
    assert len(st.widths) == 8 and st.generation == 2
    assert st.latency() == LATENCY_CFG4
    t = 1500
    assert _brute_ready(st, t * 512 + LATENCY_CFG4) == t + 1 and _brute_ready(st, t * 512 + LATENCY_CFG4 - 1) == t


def test_library_push_plan(monkeypatch):
    """The library's plan of random pushes: same counters and frames as the host, every read-back origin at or
    after what the rings kept, no ring over its capacity, and NNAB_EINVAL for counters no stream has."""
    _install(monkeypatch)
    make, _ = CONFIGS["vqt_reflect"]
    st = StreamingPyramid(make(), 1)
    widths, hop, pad_mode = st.widths, st.hop, _C.PAD_REFLECT
    assert _C.cqt_pyramid_chunk_state_bytes(1, widths, hop, 1) == 4 * st.ring.numel()
    rng = np.random.default_rng(7)
    for sizes in ([5000], list(rng.integers(0, 400, size=40)), [1] * 300 + [0, 4000]):
        received = n_carry = frames = 0
        kept = [0] * len(widths)
        for n in sizes:
            levels, t_end = _C.cqt_pyramid_chunk_plan(received, n_carry, frames, int(n), 0, widths, hop, pad_mode)
            assert t_end == st._ready(received + n)
            for s, (r0, r1, ring, keep, fir_origin, row, _, _) in enumerate(levels):
                assert r0 == st._counts(received)[s] and r1 == st._counts(received + n)[s]
                assert r1 - keep <= ring and keep >= kept[s]
                if row >= 0:
                    assert max(fir_origin, 0) >= kept[s]
                octave_origin = frames * (hop >> s) - widths[s] // 2
                assert max(octave_origin, 0) >= kept[s] or t_end == frames
                kept[s] = keep
            received += int(n)
            frames = t_end
            n_carry = st._n_carry(received, frames)
        levels, t_end = _C.cqt_pyramid_chunk_plan(received, n_carry, frames, 0, 1, widths, hop, pad_mode)
        assert levels[-1][1] > 0
    with pytest.raises(RuntimeError, match="invalid|argument|EINVAL|status -1"):
        _C.cqt_pyramid_chunk_plan(100, 5, 0, 10, 0, widths, hop, pad_mode)  # n_carry no stream has
    with pytest.raises(RuntimeError):
        _C.cqt_pyramid_chunk_plan(5000, st._n_carry(5000, 0), 0, 10, 0, widths, hop, pad_mode)  # frames behind


REPLAY = {
    "gen2": lambda: features.CQT2010v2(sr=22050, n_bins=36, fmin=220, hop_length=128, earlydownsample=False,
                                       verbose=False),
    "gen1": _vqt(),
    "gen1_early": lambda: features.CQT2010v2(sr=44100, n_bins=24, fmin=110, hop_length=256, verbose=False),
}


@pytest.mark.parametrize("name", sorted(REPLAY))
def test_plan_replay_float64(name, monkeypatch):
    """Replay pushes on the library's exported plan in float64: every signal holds NaN except the samples the
    plan declares held (the ring from its kept sample, then the push's new samples), each FIR stage computes
    exactly its store window [R0', R1') from that, and the result equals the whole-clip float64 levels to
    1e-12; the edge-fix windows lie inside the store windows, and the octave frames read only held samples."""
    _install(monkeypatch)
    m = REPLAY[name]()
    st = StreamingPyramid(m, 1)
    widths, hop, early = st.widths, st.hop, st.early
    pad_mode = _C.PAD_REFLECT
    firs = [m.lowpass_filter.double().reshape(-1).numpy()] * (len(widths) + (early > 1))
    if early > 1:
        firs[0] = m.early_downsample_filter.double().reshape(-1).numpy()
    factors = [early if (early > 1 and s == 0) else 2 for s in range(len(firs))]
    L = 9001
    rng = np.random.default_rng(11)
    x = rng.standard_normal(L)
    whole = [x]
    for s in range(len(firs) - 1):  # conv1d(stride d, padding 127) in float64
        src = np.concatenate([np.zeros(127), whole[-1], np.zeros(128)])
        n_out = (len(whole[-1]) - 2) // factors[s] + 1
        whole.append(np.array([np.dot(firs[s], src[factors[s] * o:factors[s] * o + 256]) for o in range(n_out)]))
    n_sig = len(whole)
    for sizes in ([L], list(np.diff(np.concatenate([[0], np.sort(rng.integers(0, L, 12)), [L]]))),
                  [0, 1, 1, 0, 1] + [613] * 14 + [L - 3 - 613 * 14]):
        held = [np.full(len(w) + 1, np.nan) for w in whole]
        received = n_carry = frames = 0
        for i, n in enumerate(list(sizes) + [None]):
            flush = n is None
            n = 0 if flush else int(n)
            levels, t_end = _C.cqt_pyramid_chunk_plan(received, n_carry, frames, n, int(flush), widths, hop,
                                                      pad_mode, early)
            held[0][received:received + n] = x[received:received + n]
            for s in range(n_sig - 1):
                r0n, r1n = levels[s + 1][0], levels[s + 1][1]
                _, r1, _, _, _, row, head_end, tail_begin = levels[s]
                if row < 0:
                    continue
                assert head_end == 0 or (row == 0 and head_end <= 64)
                assert tail_begin < 0 or (flush and r0n <= tail_begin and tail_begin >= r1n - 64)
                src = held[s]
                d, f = factors[s], firs[s]
                for o in range(r0n, r1n):
                    j = d * o + np.arange(256) - 127
                    v = np.where(j < 0, 0.0, src[np.clip(j, 0, len(src) - 1)])
                    v = np.where(j >= r1, 0.0 if flush else np.nan, v)
                    held[s + 1][o] = float(np.dot(f, v))
                got, want = held[s + 1][r0n:r1n], whole[s + 1][r0n:r1n]
                assert np.all(np.abs(got - want) <= 1e-12 * (1 + np.abs(want))), (name, sizes, i, s)
            # the octave frames of this push read held samples only
            for l, w in enumerate(widths):
                sg = l + (early > 1)
                total = levels[sg][1]
                for t in range(frames, t_end):
                    idx = np.arange(t * (hop >> l) - w // 2, t * (hop >> l) - w // 2 + w)
                    idx = np.abs(idx)
                    if flush:
                        idx = np.where(idx >= total, 2 * (total - 1) - idx, idx)
                    idx = idx[(idx >= 0) & (idx < total)]
                    assert not np.isnan(held[sg][idx]).any(), (name, sizes, i, l, t)
            if flush:
                break
            # what the rings no longer hold after the push
            for s in range(n_sig):
                held[s][:levels[s][3]] = np.nan
            received += n
            frames = t_end
            n_carry = st._n_carry(received, frames)
