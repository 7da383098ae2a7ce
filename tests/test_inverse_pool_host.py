"""CPU: the host logic of nnaudio_b200.streaming.InversePool against a float64 stand-in for the C call.

The stand-in for ``_C.istft_pool_forward`` keeps every slot's frames and returns, for each lane, the samples of
the offline inverse of the frames so far (``cpu_kernels.istft_forward``, float64 inside) that no later frame can
change: positions below the lane's frames x hop and below the shortest end its output can still have, re-derived
here rather than taken from the pool.  Seeded ragged schedules with idle slots, ends with and without ``length``
and restarts must give every completed stream the offline inverse of its own frames.  The C entry point's host
checks are called with fake pointers.
"""
import ctypes

import numpy as np
import pytest
import torch

import cpu_kernels
from nnaudio_b200 import _C, features
from nnaudio_b200.streaming import InversePool, StreamingInverse
from test_streaming_host import INVERSE, _install_inverse


def _install(monkeypatch):
    cpu_kernels.install(monkeypatch)
    shadow, calls = {}, []

    def istft_pool_forward(pool, lanes, X, A, n_max, T_max, packed, window, n_fft, hop, center):
        calls.append(len(lanes))
        assert lanes.shape[1] == len(_C.ISTFT_LANE_FIELDS)
        out = torch.zeros(A, n_max)
        off = n_fft // 2 if center else 0
        counts, t_most = [], 0
        for i, (s, r, F0, E0, T, end, length) in enumerate(lanes.tolist()):
            buf = shadow.setdefault((id(pool), s), [])
            if F0 == 0:
                buf.clear()
            assert sum(b.shape[2] for b in buf) == F0
            assert (r >= 0) == (T > 0)
            if T > 0:
                buf.append(X[r:r + 1, :, :T].double())
            t_most = max(t_most, T)
            allX = torch.cat(buf, 2)
            n = allX.shape[2]
            y = cpu_kernels.istft_forward(allX, packed, window, n_fft, hop, center,
                                          (length if length >= 0 else None) if end else None)[0]
            if not end:  # final: below n * hop and below the earliest end (the centre crop of n frames)
                ola_len = n_fft + hop * (n - 1)
                y = y[:max(min(n * hop, ola_len - off) - off, 0)]
            got = y[E0:]
            assert (i < A) == (len(got) > 0), (i, A, len(got))
            if i < A:
                out[i, :len(got)] = got
            counts.append(len(got))
        assert max(counts, default=0) == n_max and t_most == T_max
        return out

    monkeypatch.setattr(_C, "istft_pool_forward", istft_pool_forward)
    return calls


def _offline(m, X, onesided, length):
    if isinstance(m, features.STFT):
        return m.inverse(X, onesided=onesided, length=length)
    return m(X, onesided=onesided, length=length)


def run_schedule(pool, f_in, seed, steps=50, nan_fill=True):
    """Seeded ragged pushes: a random subset of slots in random row order, 0..t frames each, about a fifth of
    the slots idle, ends with length None / inside the span / past its end, restarts two pushes later.  Returns
    (frames, length, samples) of every completed stream."""
    S = pool.slots
    rng = np.random.default_rng(seed)
    gen = torch.Generator().manual_seed(seed)
    frames = [[] for _ in range(S)]
    got = [[] for _ in range(S)]
    ended, since = np.zeros(S, bool), np.zeros(S, int)
    done = []
    for step in range(steps + 1):
        last = step == steps
        restart = np.flatnonzero(ended & (since >= 2))
        if len(restart):
            pool.reset(restart)
            ended[restart] = False
            for s in restart:
                frames[s], got[s] = [], []
        t = int(rng.integers(1, 9))
        live = np.flatnonzero(~ended & (rng.random(S) < 0.8)) if not last else np.zeros(0, int)
        rows = rng.permutation(live)
        counts = rng.integers(0, t + 1, size=len(rows))
        if step % 7 == 3 and len(rows):
            counts[0] = t  # a long packet while others bring one frame or none
        X = torch.randn(len(rows), f_in, t, 2, generator=gen)
        for r, c in enumerate(counts):
            if nan_fill:
                X[r, :, c:] = float("nan")  # never read
        total = np.array([sum(f.shape[2] for f in frames[s]) for s in range(S)])
        added = np.zeros(S, int)
        added[rows] = counts
        have = total + added
        end = ~ended & (have > 0) & ((rng.random(S) < 0.1) | last)
        length = np.full(S, -1)
        for s in np.flatnonzero(end):
            k = rng.integers(3)
            ola = pool.n_fft + pool.hop * (have[s] - 1)
            length[s] = -1 if k == 0 else (int(rng.integers(ola // 2, ola)) if k == 1 else ola + 50)
        # a length shorter than what was returned would raise: keep it at least that long
        length = np.where((length >= 0) & (length < pool.emitted), pool.emitted, length)
        out = pool.push(X, rows, counts, end, length)
        assert out.samples.shape == (len(out.slots), int(out.counts.max()) if len(out.slots) else 0)
        assert out.slots.tolist() == sorted(out.slots.tolist())
        for i, (s, c) in enumerate(zip(out.slots.tolist(), out.counts.tolist())):
            assert c > 0 and (out.samples[i, c:] == 0).all(), "rows past their counts are exact zeros"
            got[s].append(out.samples[i, :c])
        for r, s in enumerate(rows):
            frames[s].append(X[r:r + 1, :, :counts[r]])
        for s in np.flatnonzero(end):
            done.append((torch.cat(frames[s], 2), None if length[s] < 0 else int(length[s]),
                         torch.cat(got[s]) if got[s] else torch.zeros(0)))
        ended |= end
        since = np.where(end, 0, since + 1)
    return done


@pytest.mark.parametrize("name", sorted(INVERSE))
def test_ragged_schedule_gives_every_stream_its_offline_inverse(name, monkeypatch):
    calls = _install(monkeypatch)
    make, onesided = INVERSE[name]
    m = make()
    f_in = 33 if onesided else 64
    pool = InversePool(m, 6, onesided=onesided)
    done = run_schedule(pool, f_in, seed=len(name) * 11)
    assert len(done) >= 8 and len(calls) > 0
    lengths = {None if ln is None else (ln > m.n_fft + m.stride * (X.shape[2] - 1)) for X, ln, _ in done}
    assert lengths >= {None, False, True}, "ends with length None, inside the span and past its end"
    for X, length, got in done:
        ref = _offline(m, X, onesided, length)[0]
        assert got.shape == ref.shape, (name, got.shape, ref.shape)
        assert (got - ref).abs().max().item() <= 1e-6 * ref.abs().max().item(), name


def test_pool_slots_match_one_streaming_inverse_each(monkeypatch):
    """The same frame packets through a one-stream StreamingInverse give the same samples, push by push."""
    _install(monkeypatch)
    _install_inverse(monkeypatch)
    m = features.iSTFT(n_fft=64, hop_length=16, verbose=False)
    pool = InversePool(m, 3, onesided=True)
    one = [StreamingInverse(m, 1, onesided=True) for _ in range(3)]
    rng = np.random.default_rng(4)
    X = torch.randn(3, 33, 60, 2)
    pos = np.zeros(3, int)
    while (pos < 60).any():
        counts = np.minimum(rng.integers(0, 6, size=3), 60 - pos)
        end = (pos < 60) & (pos + counts >= 60)
        rows = np.flatnonzero(counts)
        t = int(counts.max())
        Xp = torch.full((len(rows), 33, t, 2), float("nan"))
        for r, s in enumerate(rows):
            Xp[r, :, :counts[s]] = X[s, :, pos[s]:pos[s] + counts[s]]
        out = pool.push(Xp, rows, counts[rows], end)
        got = dict(zip(out.slots.tolist(), range(len(out.slots))))
        for s in range(3):
            if pos[s] >= 60:
                assert s not in got
                continue
            ref = one[s].push(X[s:s + 1, :, pos[s]:pos[s] + counts[s]])
            if end[s]:
                ref = torch.cat([ref, one[s].flush()], 1)
            if ref.shape[1]:
                i = got[s]
                assert out.counts[i] == ref.shape[1]
                assert torch.allclose(out.samples[i:i + 1, :ref.shape[1]], ref, rtol=0,
                                      atol=1e-6 * ref.abs().max().item())
            else:
                assert s not in got
        pos += counts


def test_rules_and_errors_change_nothing(monkeypatch):
    calls = _install(monkeypatch)
    m = features.iSTFT(n_fft=64, hop_length=16, verbose=False)
    with pytest.raises(TypeError):
        InversePool(features.STFT(n_fft=64, hop_length=16, verbose=False), 2)  # no iSTFT=True
    with pytest.raises(ValueError):
        InversePool(m, _C.MAX_BATCH + 1)
    with pytest.raises(ValueError):
        InversePool(features.iSTFT(n_fft=64, hop_length=80, verbose=False), 2)  # frames that do not overlap
    pool = InversePool(m, 4, onesided=True)
    assert InversePool(features.STFT(n_fft=64, hop_length=16, iSTFT=True, verbose=False), 1).onesided
    X = torch.randn(2, 33, 5, 2)
    pool.push(X, [0, 2], [5, 3])

    def state():
        return pool.frames.copy(), pool.emitted.copy(), pool.ended.copy(), len(calls)

    s0 = state()
    with pytest.raises(ValueError, match="slot 1"):
        pool.push(X, [1, 1], [1, 1])  # a slot in two rows
    with pytest.raises(ValueError, match="slot"):
        pool.push(X, [0, 4], [1, 1])  # out of range
    with pytest.raises(ValueError, match="slot 3"):
        pool.push(X, [1, 3], [1, 6])  # counts above t
    with pytest.raises(ValueError, match="slot 1"):
        pool.push(X, [1, 3], [-1, 0])
    with pytest.raises(ValueError):
        pool.push(torch.randn(2, 64, 5, 2), [0, 1], [1, 1])  # bins of a two-sided spectrum
    with pytest.raises(ValueError):
        pool.push(X.double(), [0, 1], [1, 1])
    with pytest.raises(ValueError):
        pool.push(X, [0], [1])  # one slot per row
    with pytest.raises(NotImplementedError):
        pool.push(X.clone().requires_grad_(), [0, 1], [1, 1])
    with pytest.raises(TypeError):
        pool.push(X, [0.5, 1], [1, 1])
    with pytest.raises(TypeError):
        pool.push(X, torch.tensor([0, 1], device="meta"), [1, 1])  # row slots stay on the CPU
    with pytest.raises(TypeError):
        pool.push(X, [0, 1], torch.tensor([1, 1], device="meta"))
    with pytest.raises(TypeError):
        pool.push(X, [0, 1], [1, 1], torch.zeros(4, dtype=torch.bool, device="meta"))
    with pytest.raises(TypeError):
        pool.push(X, [0, 1], [1, 1], [True, False, False, False], torch.zeros(4, dtype=torch.int64, device="meta"))
    with pytest.raises(RuntimeError, match="slot 1"):
        pool.push(X[:1], [0], [1], [False, True, False, False])  # slot 1 never had a frame
    with pytest.raises(ValueError, match="slot 0"):
        pool.push(X[:0], [], [], [True, False, False, False], [10, -1, -1, -1])  # shorter than returned
    assert all(np.array_equal(a, b) for a, b in zip(state()[:3], s0[:3])) and state()[3] == s0[3]
    out = pool.push(X[:0], [], [], [True, False, False, False])
    # 5 frames: positions [32, 80) returned; the end returns the rest of the centre crop, [80, 96)
    assert out.slots.tolist() == [0] and out.counts.tolist() == [96 - 80]
    with pytest.raises(RuntimeError, match="slot 0"):
        pool.push(X[:1], [0], [1])  # an ended slot takes nothing ...
    with pytest.raises(RuntimeError, match="slot 0"):
        pool.push(X[:0], [], [], [True, False, False, False])  # ... and no second end
    out = pool.push(X[:0], [], [])  # an empty push
    assert out.samples.shape == (0, 0) and out.slots.numel() == 0
    out = pool.push(X, [1, 3], [0, 1])  # one frame: nothing final yet, and a row with no frames
    assert out.slots.numel() == 0 and pool.frames.tolist() == [5, 0, 3, 1]
    pool.reset([0])
    assert pool.frames[0] == 0 and pool.emitted[0] == 0 and not pool.ended[0] and pool.frames[2] == 3
    assert pool.push(X[:1], [0], [4]).counts.tolist() == [4 * 16 - 32]


def test_stream_pool_output_feeds_the_inverse_pool(monkeypatch):
    """StreamPool -> InversePool with each slot's length set to its sample count reconstructs the waveform."""
    _install(monkeypatch)
    import test_stream_pool_host as sp
    sp._install(monkeypatch, "fused")
    stft = features.STFT(n_fft=64, hop_length=16, output_format="Complex", iSTFT=True, verbose=False)
    fwd, inv = sp.StreamPool(stft, 3), InversePool(stft, 3)
    rng = np.random.default_rng(9)
    x = torch.randn(3, 700)
    pos, parts = np.zeros(3, int), [[] for _ in range(3)]
    while (pos < 700).any():
        lengths = np.minimum(rng.integers(0, 120, size=3), 700 - pos)
        end = (pos < 700) & (pos + lengths >= 700)
        chunk = torch.zeros(3, int(lengths.max()))
        for s in range(3):
            chunk[s, :lengths[s]] = x[s, pos[s]:pos[s] + lengths[s]]
        a = fwd.push(chunk, lengths, end)
        y = inv.push(a.frames.float(), a.slots, a.counts, end, np.where(end, 700, -1))
        for i, (s, c) in enumerate(zip(y.slots.tolist(), y.counts.tolist())):
            parts[s].append(y.samples[i, :c])
        pos += lengths
    for s in range(3):
        assert np.allclose(x[s].numpy(), torch.cat(parts[s]).numpy(), rtol=1e-5, atol=1e-3)


# ------------------------------------------------------------------------------------------- C host checks
EINVAL = -1


def _lanes(*rows):
    flat = [int(v) for r in rows for v in r]
    return (ctypes.c_int64 * max(len(flat), 1))(*flat)


def _call(lanes, n_lanes, A, n_max, T_max, R=3, t=4, slots=4, X=256, out=256, hop=16):
    P = ctypes.c_void_p
    p = P(256)  # never dereferenced on the host
    return _C.lib().nnab_istft_pool_forward(p, lanes, p, n_lanes, A, slots, None if X is None else P(X), R, 33, t, p,
                                            p, 64, hop, 1, None if out is None else P(out), n_max, T_max, None, 0,
                                            None)


def test_istft_pool_entry_point_rejects_bad_lane_tables_on_the_host():
    # n_fft 64, hop 16, centred: a new stream's first 4 frames make positions [32, 64) final (32 samples), one
    # frame makes none
    fresh = lambda s, r, T=4, end=0, length=-1: (s, r, 0, 0, T, end, length)  # noqa: E731
    ok = _call(_lanes(fresh(0, 0), fresh(2, 1, 1)), 2, 1, 32, 4)
    assert ok != EINVAL, "a valid table passes the checks (and stops at the device or the workspace)"
    assert ok in (-3, -4, -5)
    assert _call(_lanes(fresh(0, 0), fresh(2, 1, 1)), 2, 1, 31, 4) == EINVAL, "n_max is the longest row's count"
    assert _call(_lanes(fresh(0, 0), fresh(2, 1, 1)), 2, 1, 32, 3) == EINVAL, "T_max is the most frames of a lane"
    assert _call(_lanes(fresh(0, 0), fresh(2, 1, 1)), 2, 2, 32, 4) == EINVAL, "A counts the lanes with samples"
    assert _call(_lanes(fresh(2, 1, 1), fresh(0, 0)), 2, 1, 32, 4) == EINVAL, "the lanes with samples come first"
    assert _call(_lanes(fresh(2, 0), fresh(0, 1)), 2, 2, 32, 4) == EINVAL, "slots ascend within a group"
    assert _call(_lanes(fresh(0, 0), fresh(0, 1)), 2, 2, 32, 4) == EINVAL, "a slot appears once"
    assert _call(_lanes(fresh(0, 0), fresh(1, 0)), 2, 2, 32, 4) == EINVAL, "a row feeds one lane"
    assert _call(_lanes(fresh(4, 0)), 1, 1, 32, 4) == EINVAL, "slot out of range"
    assert _call(_lanes(fresh(0, 3)), 1, 1, 32, 4) == EINVAL, "row out of range"
    assert _call(_lanes(fresh(0, -1)), 1, 1, 32, 4) == EINVAL, "a lane with frames has a row"
    assert _call(_lanes((0, 0, 4, 32, 0, 1, -1)), 1, 1, 48, 0) == EINVAL, "a lane without frames has row -1"
    assert _call(_lanes(fresh(0, 0)), 1, 1, 32, 4, t=3) == EINVAL, "T <= t"
    assert _call(_lanes(fresh(0, 0, 0)), 1, 0, 0, 0) == EINVAL, "a lane with nothing to do"
    assert _call(_lanes(fresh(0, 0, 4, 2)), 1, 1, 32, 4) == EINVAL, "end is 0 or 1"
    assert _call(_lanes((0, -1, 4, 3, 0, 1, -1)), 1, 1, 45, 0) == EINVAL, "counters no stream has"
    assert _call(_lanes((0, -1, 4, 32, 0, 1, 10)), 1, 0, 0, 0) == EINVAL, "length shorter than returned"
    assert _call(_lanes(fresh(0, -1, 0, 1)), 1, 0, 0, 0) == EINVAL, "an end without any frame"
    assert _call(_lanes(fresh(0, 0)), 1, 1, 32, 4, hop=65) == EINVAL, "frames that do not overlap"
    assert _call(_lanes(fresh(0, 0)), 1, 1, 32, 4, X=None) == EINVAL, "no frames"
    assert _call(_lanes(fresh(0, 0)), 1, 1, 32, 4, out=None) == EINVAL, "no output"
    assert _call(None, 1, 1, 32, 4) == EINVAL, "no host table"
    assert _call(_lanes(fresh(0, 0)), 1, 1, 32, 4, slots=0) == EINVAL
    assert _call(_lanes(fresh(0, 0), fresh(1, 1)), 2, 2, 32, 4, slots=1) == EINVAL, "more lanes than slots"
    # an end with no new frames and length None returns the rest of 4 frames' centre crop: positions [64, 80)
    assert _call(_lanes((0, -1, 4, 32, 0, 1, -1)), 1, 1, 16, 0) != EINVAL


def test_istft_pool_workspace_query_obeys_its_rule():
    lib = _C.lib()
    up = lambda v, a: (v + a - 1) // a * a  # noqa: E731
    assert lib.nnab_istft_pool_workspace_bytes(0, 33, 5, 64, 16) == 0
    for n_lanes, f_in, T_max, n_fft, hop in ((1, 33, 0, 64, 16), (3, 33, 5, 64, 16), (256, 257, 4, 512, 128),
                                             (7, 101, 9, 200, 100), (5, 1025, 1, 2048, 512)):
        lead = up(n_lanes * up(n_fft, 8) * 4, 256)  # n_lanes rows of n_fft floats, rows rounded up to 8 floats
        assert lib.nnab_istft_pool_workspace_bytes(n_lanes, f_in, T_max, n_fft, hop) == \
            lib.nnab_istft_workspace_bytes(n_lanes, f_in, max(T_max, 1), n_fft, hop) + lead


def test_istft_chunk_workspace_equals_pool_of_its_lanes():
    """A lock-step inverse push of B streams is a pool push of B lanes that share its counters, lane b in slot b
    and X row b: its workspace query equals the pool's for n_lanes = B and T_max = T, over seeded cases."""
    lib = _C.lib()
    rng = np.random.default_rng(5)
    for _ in range(200):
        n_fft = int(rng.choice([16, 64, 200, 512, 2048]))
        hop = int(rng.integers(1, n_fft + 1))
        f_in = int(rng.choice([n_fft // 2 + 1, n_fft]))
        T, B = int(rng.integers(0, 40)), int(rng.choice([1, 2, 7, 256, 65535]))
        assert lib.nnab_istft_chunk_workspace_bytes(B, f_in, T, n_fft, hop) == \
            lib.nnab_istft_pool_workspace_bytes(B, f_in, T, n_fft, hop), (B, f_in, T, n_fft, hop)
