"""CPU: the plan of the device pyramid pool (``nnab_debug_device_pyramid_plan``, the per-slot function its plan launch
runs) against PyramidPool's numpy bookkeeping, and its fixed geometry (``nnab_cqt_pyramid_pool_device_caps``)
against a brute-force maximum.

Seeded traces with idle slots, zero-length pushes, ends, restarts, out-of-range lengths, pushes after an end and ends
on streams too short for the module: every tick, each slot's lane, count and counters must be those PyramidPool
computes for it, a refused slot must get the error code of the exception PyramidPool raises for that slot alone (and
``check()`` that exception), and every other slot a lane that returns nothing.  The zero lane of an idle slot maps
to no frame, no FIR row, no carry and no edge fix.  The caps equal the largest frame count, FIR output count and
carry over every push of at most ``chunk`` samples on a long range of stream positions, computed here from the
streaming rules in numpy; no push without an end is ever refused on those ranges.
"""
import copy

import numpy as np
import pytest
import torch

from nnaudio_b200 import _C, features
from nnaudio_b200.streaming import DevicePyramidPool, PyramidPool
from test_pyramid_pool_host import _install
from test_streaming_pyramid_host import REPLAY, _vqt

TRACES = {
    "gen2": REPLAY["gen2"],
    "gen1": REPLAY["gen1"],
    "gen1_early": REPLAY["gen1_early"],
    "vqt_gamma5": lambda: features.VQT(sr=8000, n_bins=36, fmin=55, gamma=5, hop_length=64, earlydownsample=False,
                                       verbose=False),
    "vqt_constant": _vqt(pad_mode="constant"),
}


def _host_pool(m, S):
    """PyramidPool's bookkeeping with the C call replaced by a recorder."""
    p = PyramidPool(m, S)
    p.rec = []
    p._advance = lambda chunk, lanes, A, T_max, count: p.rec.append((lanes.copy(), count.copy()))
    return p


def _alone(host):
    """A copy of the host pool's counters whose pushes record nothing."""
    c = copy.copy(host)
    c.received, c.frames, c.ended = host.received.copy(), host.frames.copy(), host.ended.copy()
    c._advance = lambda *a: None
    return c


def _raises(fn):
    try:
        fn()
    except Exception as e:
        return e
    return None


@pytest.mark.parametrize("name", sorted(TRACES))
def test_plan_matches_pyramid_pool(name, monkeypatch):
    _install(monkeypatch)
    m = TRACES[name]()
    S, chunk = 9, 700
    host = _host_pool(m, S)
    pad_mode = _C.PAD_REFLECT if m.pad_mode == "reflect" else _C.PAD_CONSTANT
    widths, hop, early = host.widths, host.hop, host.early
    counters = np.zeros((3, S), np.int64)
    errors, info = np.zeros(S, np.int32), np.zeros((S, 2), np.int64)
    sticky = np.zeros(S, np.int32)
    rng = np.random.default_rng(len(name))
    x = torch.zeros(S, chunk)
    codes_seen, ends = set(), 0
    for step in range(160):
        restart = (rng.random(S) < 0.04) | (host.ended & (rng.random(S) < 0.3))
        if restart.any():
            host.reset(np.flatnonzero(restart))
            counters[:, restart] = 0
            errors[restart], info[restart], sticky[restart] = 0, 0, 0
        lengths = rng.choice([0, 1, hop - 1, hop, chunk], size=S) if step % 3 == 0 else rng.integers(0, chunk + 1, S)
        lengths = lengths * (rng.random(S) < 0.85)
        end = rng.random(S) < 0.08
        bad = rng.random(S) < 0.03
        lengths = np.where(bad, rng.choice([-1, chunk + 1, chunk + 50], size=S), lengths)
        # PyramidPool on every slot alone: what it raises, if anything
        expect = np.zeros(S, np.int32)
        excs = {}
        for s in range(S):
            ln, en = np.zeros(S, np.int64), np.zeros(S, bool)
            ln[s], en[s] = lengths[s], end[s]
            with torch.no_grad():
                e = _raises(lambda: _alone(host).push(x, ln, en))
            if e is not None:
                excs[s] = e
                expect[s] = (_C.LANE_ELENGTH if isinstance(e, ValueError) and "chunk width" in str(e) else
                             _C.LANE_EENDED if "has ended" in str(e) else _C.LANE_ESHORT)
        ok = expect == 0
        ends += int((end & ok).sum())
        host.rec.clear()
        host.push(x, np.where(ok, lengths, 0), end & ok)
        lanes, counts = _C.debug_device_pyramid_plan(counters, lengths.astype(np.int32), end, errors, info, chunk,
                                                     widths, hop, early, pad_mode)
        want_lanes = np.zeros((S, 6), np.int64)
        want_lanes[:, 0] = np.arange(S)
        want_counts = np.zeros(S, np.int64)
        if host.rec:
            h_lanes, h_count = host.rec[0]
            want_lanes[h_lanes[:, 0]] = h_lanes
            want_counts[h_lanes[:, 0]] = h_count
        assert (lanes == want_lanes).all(), (step, lanes, want_lanes)
        assert (counts == want_counts).all(), step
        assert (counters[0] == host.received).all() and (counters[1] == host.frames).all()
        assert (counters[2] == host.ended).all()
        fresh = sticky == 0
        sticky = np.where(sticky != 0, sticky, expect)
        assert (errors == sticky).all(), (step, errors, sticky)
        for s, e in excs.items():  # check() of a pool whose only error is this one raises PyramidPool's exception
            if not fresh[s]:
                continue
            codes_seen.add(int(expect[s]))
            assert info[s, 0] == (host.received[s] + lengths[s] if expect[s] == _C.LANE_ESHORT else lengths[s])
            only = np.zeros(S, np.int32)
            only[s] = errors[s]
            view = DevicePyramidPool.__new__(DevicePyramidPool)
            view.slots, view.chunk, view.module = S, chunk, m
            view.errors, view.error_info = torch.from_numpy(only), torch.from_numpy(info.copy())
            with pytest.raises(type(e)) as got:
                view.check()
            assert str(got.value) == str(e), (got.value, e)
    assert codes_seen == {_C.LANE_ELENGTH, _C.LANE_EENDED, _C.LANE_ESHORT}, codes_seen
    assert ends >= 5


def test_zero_lane_maps_to_nothing(monkeypatch):
    """An idle, ended or dropped slot's all-zero lane: no frame, no FIR row, no carry, no edge fix, and (reflect
    padding) an octave origin of -pad whose mirror the split kernel reads as zeros."""
    _install(monkeypatch)
    for name in ("gen2", "gen1_early"):
        pool = PyramidPool(REPLAY[name](), 1)
        zero = np.zeros((1, 6), np.int64)
        # the device plan of one idle slot
        counters = np.zeros((3, 1), np.int64)
        errors, info = np.zeros(1, np.int32), np.zeros((1, 2), np.int64)
        lanes, counts = _C.debug_device_pyramid_plan(counters, np.zeros(1, np.int32), np.zeros(1, bool), errors, info,
                                                     64, pool.widths, pool.hop, pool.early, _C.PAD_REFLECT)
        assert (lanes == zero).all() and counts[0] == 0 and not counters.any() and not errors.any()
        # its (signal, lane) descriptors, by the chunk plan's rules: the push of nothing
        sigs, t_end = _C.cqt_pyramid_chunk_plan(0, 0, 0, 0, 0, pool.widths, pool.hop, _C.PAD_REFLECT, pool.early)
        assert t_end == 0
        for r0, r1, _, keep, _, t0, head, tail in sigs:
            assert (r0, r1, keep, t0, head, tail) == (0, 0, 0, -1, 0, -1)


# ---- the fixed geometry ----------------------------------------------------------------------------------------- #
class _Rules:
    """The streaming rules of a pyramid (StreamingPyramid / PyramidPool), vectorised over stream positions."""

    def __init__(self, widths, hop, early, reflect):
        self.widths, self.hop, self.early, self.reflect = list(widths), hop, early, reflect
        self.gen2 = early == 1 and all(w // 2 == 128 for w in widths[:-1])
        self.c = 130 if self.gen2 else 129
        self.e = 1 if early > 1 else 0
        self.d = [early if (self.e and s == 0) else 2 for s in range(len(widths) + self.e - 1)]

    def counts(self, raw, end):
        R = [raw]
        for d in self.d:
            r = R[-1]
            R.append(np.where(r < 2, 0, (r - 2) // d + 1) if end else np.where(r >= self.c, (r - self.c) // d + 1, 0))
        return R

    def ready(self, R):
        t = None
        for i, w in enumerate(self.widths):
            r, pad, h = R[i + self.e], w // 2, self.hop >> i
            f = np.where(r < w - pad, 0, (r - (w - pad)) // h + 1)
            if self.reflect:
                f = np.where(r < pad + 1, 0, f)
            t = f if t is None else np.minimum(t, f)
        return t

    def end_frames(self, R):
        """(frames, accepted) at an end: every level non-empty, equal octave frame counts, at least one."""
        fs = []
        ok = np.ones(R[0].shape, bool)
        for i, w in enumerate(self.widths):
            r = R[i + self.e]
            span = r + 2 * (w // 2) - w
            f = np.where(span < 0, 0, span // (self.hop >> i) + 1)
            ok &= (r > 0) & (f > 0)
            fs.append(f)
        for f in fs[1:]:
            ok &= f == fs[0]
        return fs[0], ok

    def keep(self, R, frames, s):
        k = R[s]
        l = s - self.e
        if l >= 0:
            pad, h = self.widths[l] // 2, self.hop >> l
            st = frames * h - pad
            if pad > 0:
                st = np.minimum(st, R[s] - (pad + 1))
            k = np.minimum(np.maximum(st, 0), R[s])
        if s + 1 < len(R):
            k = np.minimum(k, np.maximum(0, 128 * self.d[s] * (R[s + 1] // 128) - 128))
        return k

    def push(self, rec, n, end):
        """(count, per-stage FIR outputs from the first row, per-signal carry, accepted) of the pushes of n samples
        from positions rec (no end: ring capacity is not modelled, the caps query checks it)."""
        R0 = self.counts(rec, False)
        frames = self.ready(R0)
        R1 = self.counts(rec + n, end)
        if end:
            t_end, ok = self.end_frames(R1)
            ok &= t_end >= frames
        else:
            t_end, ok = self.ready(R1), np.ones(rec.shape, bool)
        count = np.where(ok, t_end - frames, 0)
        fir = [np.where(ok & (R1[s + 1] > R0[s + 1]), R1[s + 1] - 128 * (R0[s + 1] // 128), 0)
               for s in range(len(R0) - 1)] + [np.zeros(rec.shape, np.int64)]
        carry = [np.zeros(rec.shape, np.int64) if end else R1[s] - np.maximum(self.keep(R1, t_end, s), R0[s])
                 for s in range(len(R0))]
        return count, fir, carry, ok


def _window_max(a, w):
    """out[i] = a[i:i + w].max() for every full window."""
    k, m = 1, a
    while 2 * k <= w:
        m = np.maximum(m[:-k], m[k:])  # m[i] = a[i:i + 2k].max()
        k *= 2
    n = len(a) - w + 1
    return np.maximum(m[:n], m[w - k:w - k + n])


def _brute(rules, chunk, rec_max, carry_recs=None):
    """The caps by brute force over every push of n in [0, chunk] samples from received in [0, rec_max), with and
    without an end.  Frames and FIR outputs: a push's value is a nondecreasing function of a quantity of its total
    t = received + n (the frame bound, R1 of the next signal) less one of its start, so the sliding maximum over t
    in [received, received + chunk] is the maximum over n (at an end over the accepted totals, whose frame bound and
    counts grow with t).  Carries push by push over every n on `carry_recs` (default: every position)."""
    rec = np.arange(rec_max, dtype=np.int64)
    t = np.arange(rec_max + chunk, dtype=np.int64)
    n_sig = len(rules.widths) + rules.e
    R0 = rules.counts(rec, False)
    frames = rules.ready(R0)
    T_cap, fir_cap = 0, [0] * n_sig
    # without an end
    R1 = rules.counts(t, False)
    T_cap = max(T_cap, int((_window_max(rules.ready(R1), chunk + 1) - frames).max()))
    for s in range(n_sig - 1):
        top = _window_max(R1[s + 1], chunk + 1)
        fir_cap[s] = max(fir_cap[s], int(np.where(top > R0[s + 1], top - 128 * (R0[s + 1] // 128), 0).max()))
    # at an end: the last accepted total of the window, if its frame bound reaches the frames returned
    R1 = rules.counts(t, True)
    t_end, ok = rules.end_frames(R1)
    last = _window_max(np.where(ok, t, -1), chunk + 1)
    live = (last >= 0) & (t_end[np.maximum(last, 0)] >= frames)
    if live.any():
        T_cap = max(T_cap, int((t_end[last[live]] - frames[live]).max()))
        for s in range(n_sig - 1):
            top, r0 = R1[s + 1][last[live]], R0[s + 1][live]
            fir_cap[s] = max(fir_cap[s], int(np.where(top > r0, top - 128 * (r0 // 128), 0).max()))
    carry_cap = [0] * n_sig
    r = rec if carry_recs is None else carry_recs
    for n in range(chunk + 1):
        _, _, carry, _ = rules.push(r, n, False)
        carry_cap = [max(a, int(b.max())) for a, b in zip(carry_cap, carry)]
    return T_cap, fir_cap, carry_cap


SYNTHETIC = {  # (widths, hop, early, pad_mode): small pyramids whose start-up and period are short
    "gen2_3oct": ([256, 256, 64], 8, 1, _C.PAD_REFLECT),
    "gen1_3oct": ([32, 24, 16], 8, 1, _C.PAD_REFLECT),
    "gen1_constant": ([32, 24, 16], 4, 1, _C.PAD_CONSTANT),
    "gen1_early": ([16, 16], 4, 4, _C.PAD_REFLECT),
}


@pytest.mark.parametrize("name", sorted(SYNTHETIC))
def test_caps_equal_brute_force_small(name):
    widths, hop, early, pm = SYNTHETIC[name]
    rules = _Rules(widths, hop, early, pm == _C.PAD_REFLECT)
    for chunk in (1, 37, 130):
        got = _C.cqt_pyramid_pool_device_caps(chunk, widths, hop, early, pm)
        want = _brute(rules, chunk, 40000)
        assert got == want, (name, chunk, got, want)


def test_caps_equal_brute_force_cfg4():
    """cfg4 (CQT2010v2, 88 bins at 22.05 kHz, hop 512, 8 octaves, generation 2) at 10 and 40 ms chunks.  Frames and
    FIR outputs over every n and 400 k stream positions; carries over every n on the first 3000 positions and one
    whole period past start-up (the rest at n = chunk)."""
    rules_w = [256] * 8  # cfg4's bank widths (test_streaming_pyramid_host: 8 octaves, generation 2)
    rules = _Rules(rules_w, 512, 1, True)
    for chunk in (220, 882):
        got = _C.cqt_pyramid_pool_device_caps(chunk, rules_w, 512, 1, _C.PAD_REFLECT)
        period = 128 * 128
        late = np.arange(170000, 170000 + period + chunk, dtype=np.int64)
        recs = np.concatenate([np.arange(3000, dtype=np.int64), late])
        want = _brute(rules, chunk, 400000, carry_recs=recs)
        _, _, tail, _ = rules.push(np.arange(400000, dtype=np.int64), chunk, False)
        want = (want[0], want[1], [max(a, int(b.max())) for a, b in zip(want[2], tail)])
        assert got == want, (chunk, got, want)
        # the look-ahead an end returns: about 32640 / 512 frames plus the chunk's own
        assert 60 <= got[0] <= 66 + chunk // 512, got[0]


def test_no_refusal_without_an_end():
    """Every push of at most `chunk` samples without an end passes the one-stream rules (the ring bounds), on the
    small pyramids and the cfg4 geometry over long ranges of positions, through the device plan itself."""
    for widths, hop, early, pm in list(SYNTHETIC.values()) + [([256] * 8, 512, 1, _C.PAD_REFLECT)]:
        rules = _Rules(widths, hop, early, pm == _C.PAD_REFLECT)
        rec = np.arange(0, 200000, 7, dtype=np.int64)
        frames = rules.ready(rules.counts(rec, False))
        for n in (1, 130, 882):
            counters = np.stack([rec, frames, np.zeros_like(rec)])
            errors, info = np.zeros(len(rec), np.int32), np.zeros((len(rec), 2), np.int64)
            _, counts = _C.debug_device_pyramid_plan(counters, np.full(len(rec), n, np.int32),
                                                     np.zeros(len(rec), bool), errors, info, 882, widths, hop, early,
                                                     pm)
            assert not errors.any(), (widths, n, np.flatnonzero(errors)[:5])
            assert (counters[0] == rec + n).all()


def test_construction_and_push_refusals_before_device_work(monkeypatch):
    _install(monkeypatch)
    m = REPLAY["gen1"]()
    with pytest.raises(ValueError):
        DevicePyramidPool(m, 0, 100)
    with pytest.raises(ValueError, match="chunk"):
        DevicePyramidPool(m, 2, 0)
    with pytest.raises(ValueError, match="dtype"):
        DevicePyramidPool(m, 2, 100, dtype=torch.float64)
    with pytest.raises(TypeError, match="StreamingPyramid"):
        DevicePyramidPool(features.STFT(n_fft=64, hop_length=16, verbose=False), 2, 100)
    with pytest.raises(ValueError, match="multiple"):
        DevicePyramidPool(features.CQT2010v2(sr=22050, n_bins=36, fmin=220, hop_length=126, earlydownsample=False,
                                             verbose=False), 2, 100)
    # push checks: a pool whose device side was never built refuses before reaching it
    pool = DevicePyramidPool.__new__(DevicePyramidPool)
    pool.slots, pool.chunk, pool.dtype, pool.ring = 2, 100, torch.float32, torch.zeros(1)
    pool._no_end = torch.zeros(2, dtype=torch.bool)
    i32 = torch.zeros(2, dtype=torch.int32)
    for x, lengths, exc in [(torch.zeros(2, 99), i32, ValueError), (torch.zeros(2, 100).half(), i32, ValueError),
                            (torch.zeros(3, 100), i32, ValueError), (torch.zeros(2, 100), i32.long(), TypeError),
                            (torch.zeros(2, 100), [0, 0], TypeError), (torch.zeros(2, 100), i32[:1], ValueError),
                            (torch.zeros(2, 100, requires_grad=True), i32, NotImplementedError)]:
        with pytest.raises(exc):
            pool.push(x, lengths)
    with pytest.raises(TypeError):
        pool.push(torch.zeros(2, 100), i32, torch.zeros(2, dtype=torch.uint8))


def test_c_entry_host_checks():
    """The device forward's host checks and queries (dummy device pointers: an EINVAL returns before any use)."""
    import ctypes
    L = _C.lib()
    widths = [256] * 8
    w = (ctypes.c_int32 * 8)(*widths)
    T_cap = _C.cqt_pyramid_pool_device_caps(882, widths, 512, 1, _C.PAD_REFLECT)[0]
    ws = L.nnab_cqt_pyramid_pool_device_workspace_bytes(64, 882, 8, w, 512, 1, _C.PAD_REFLECT)
    assert ws > 0 and ws > L.nnab_cqt_pyramid_pool_device_workspace_bytes(8, 882, 8, w, 512, 1, _C.PAD_REFLECT)
    assert L.nnab_cqt_pyramid_pool_device_workspace_bytes(64, 0, 8, w, 512, 1, _C.PAD_REFLECT) == 0
    assert L.nnab_cqt_pyramid_pool_device_workspace_bytes(64, 882, 8, w, 500, 1, _C.PAD_REFLECT) == 0
    p = ctypes.c_void_p(256)
    arr = (ctypes.c_void_p * 8)(*([256] * 8))
    EINVAL, EUNSUPPORTED = -1, _C.EUNSUPPORTED

    def call(T_max=T_cap, n=882, pitch=882, dtype=_C.DTYPE_F32, path=0, packed=arr, lengths=p):
        return L.nnab_cqt_pyramid_pool_device_forward(
            p, p, lengths, p, p, p, p, p, p, dtype, 64, n, pitch, 8, arr, arr, packed, w, 12, p, p, None, None, 1,
            512, _C.PAD_REFLECT, 88, None, 1.0, _C.FMT_MAGNITUDE, 0.0, p, T_max, p, ws, path, None)

    assert call(T_max=T_cap + 1) == EINVAL
    assert call(T_max=T_cap - 1) == EINVAL
    assert call(pitch=881) == EINVAL
    assert call(dtype=7) == EINVAL
    assert call(lengths=None) == EINVAL
    assert call(n=0, T_max=0) == EINVAL
    assert call(path=1) == EUNSUPPORTED  # the SIMT path: refused on the host, nothing enqueued
    assert call(packed=(ctypes.c_void_p * 8)(*([256] * 7 + [None]))) == EUNSUPPORTED
