"""CPU: the plan of the device pools (``nnab_debug_device_pool_plan`` / ``nnab_debug_device_istft_plan``, the
per-slot function the plan launch runs) against the numpy bookkeeping of StreamPool and InversePool.

Seeded traces with idle slots, zero-length pushes, ends, restarts and refused pushes: every tick, each slot's lane,
count and counters must be those StreamPool / InversePool compute for it, a refused slot must get the error code of
the exception the host pool raises for that slot alone (and ``check()`` that exception), and every other slot a lane
that returns nothing.  T_cap and n_cap are held to a brute-force maximum over stream positions.
"""
import copy
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from nnaudio_b200 import _C, features
from nnaudio_b200.streaming import (DeviceInversePool, DeviceStreamPool, InversePool, StreamPool, _ready_frames)

FWD = [  # (n_fft, hop, center, pad_mode)
    (512, 128, True, "reflect"),
    (512, 256, True, "constant"),
    (1024, 256, False, "reflect"),
    (400, 100, True, "reflect"),
    (255, 64, True, "reflect"),
]


def _host_stream_pool(S, stft):
    """StreamPool's bookkeeping without a device: its push with the C call replaced by a recorder."""
    p = StreamPool.__new__(StreamPool)
    p.slots, p.K, p.hop = S, stft.n_fft, stft.stride if hasattr(stft, "stride") else stft.hop_length
    p.pad = p.K // 2 if stft.center else 0
    p._reflect = p.pad > 0 and stft.pad_mode == "reflect"
    p.received, p.frames, p.ended = np.zeros(S, np.int64), np.zeros(S, np.int64), np.zeros(S, bool)
    p.dtype = None
    p._st = SimpleNamespace(_check_length=stft._check_length)
    p.rec = []
    p._advance = lambda chunk, lanes, A, T_max, count: p.rec.append((lanes.copy(), count.copy()))
    return p


def _raises(fn):
    try:
        fn()
    except Exception as e:
        return e
    return None


def _device_view(pool_cls, S, errors, info, **attrs):
    v = pool_cls.__new__(pool_cls)
    v.slots, v.errors, v.error_info = S, torch.from_numpy(errors.copy()), torch.from_numpy(info.copy())
    for k, a in attrs.items():
        setattr(v, k, a)
    return v


@pytest.mark.parametrize("cfg", FWD)
def test_forward_plan_matches_stream_pool(cfg):
    n_fft, hop, center, mode = cfg
    stft = features.STFT(n_fft=n_fft, hop_length=hop, center=center, pad_mode=mode, verbose=False)
    S, chunk = 10, 300
    host = _host_stream_pool(S, stft)
    pad_mode = _C.PAD_REFLECT if mode == "reflect" else _C.PAD_CONSTANT
    counters = np.zeros((3, S), np.int64)
    errors, info = np.zeros(S, np.int32), np.zeros((S, 2), np.int64)
    sticky = np.zeros(S, np.int32)
    rng = np.random.default_rng(n_fft + hop)
    x = torch.zeros(S, chunk)
    seen = set()
    for step in range(150):
        restart = (rng.random(S) < 0.06) | (host.ended & (rng.random(S) < 0.3))
        if restart.any():
            host.reset(np.flatnonzero(restart))
            counters[:, restart] = 0
            errors[restart], info[restart], sticky[restart] = 0, 0, 0
        lengths = rng.choice([0, 1, hop - 1, hop, chunk], size=S) if step % 3 == 0 else rng.integers(0, chunk + 1, S)
        lengths = lengths * (rng.random(S) < 0.8)
        end = rng.random(S) < 0.1
        bad = rng.random(S) < 0.03
        lengths = np.where(bad, rng.choice([-1, chunk + 1, chunk + 50], size=S), lengths)
        # the host pool on every slot alone: what it raises, if anything
        expect = np.zeros(S, np.int32)
        excs = {}
        for s in range(S):
            ln, en = np.zeros(S, np.int64), np.zeros(S, bool)
            ln[s], en[s] = lengths[s], end[s]
            e = _raises(lambda: copy.deepcopy(host).push(x, ln, en))
            if e is not None:
                excs[s] = e
                expect[s] = (_C.LANE_ELENGTH if isinstance(e, ValueError) and "chunk width" in str(e) else
                             _C.LANE_EENDED if "has ended" in str(e) else _C.LANE_ESHORT)
        ok = expect == 0
        host.rec.clear()
        host.push(x, np.where(ok, lengths, 0), end & ok)
        lanes, counts = _C.debug_device_pool_plan(counters, lengths.astype(np.int32), end, errors, info, chunk,
                                                  n_fft, hop, host.pad, pad_mode)
        want_lanes = np.zeros((S, 6), np.int64)
        want_lanes[:, 0] = np.arange(S)
        want_counts = np.zeros(S, np.int64)
        h_lanes, h_count = host.rec[0]
        want_lanes[h_lanes[:, 0]] = h_lanes
        want_counts[h_lanes[:, 0]] = h_count
        assert (lanes == want_lanes).all(), (step, lanes, want_lanes)
        assert (counts == want_counts).all(), step
        assert (counters[0] == host.received).all() and (counters[1] == host.frames).all()
        assert (counters[2] == host.ended).all()
        fresh = sticky == 0  # slots whose code and values are this push's
        sticky = np.where(sticky != 0, sticky, expect)
        assert (errors == sticky).all(), (step, errors, sticky)
        for s, e in excs.items():  # check() of a pool whose only error is this one raises the host's exception
            if not fresh[s] or expect[s] in seen and expect[s] != _C.LANE_ESHORT:
                continue
            seen.add(expect[s])
            only = np.zeros(S, np.int32)
            only[s] = errors[s]
            view = _device_view(DeviceStreamPool, S, only, info, chunk=chunk, _st=host._st)
            with pytest.raises(type(e)) as got:
                view.check()
            assert str(got.value) == str(e), (got.value, e)
    short_possible = (host.pad > 0 and host._reflect) or 2 * host.pad < n_fft  # else every end has a frame
    assert seen >= {_C.LANE_ELENGTH, _C.LANE_EENDED} | ({_C.LANE_ESHORT} if short_possible else set()), seen


def _host_inverse_pool(S, n_fft, hop, center):
    p = InversePool.__new__(InversePool)
    p.slots, p.n_fft, p.hop, p.center = S, n_fft, hop, center
    p.f_in, p.offset = n_fft // 2 + 1, n_fft // 2 if center else 0
    p.frames, p.emitted, p.ended = np.zeros(S, np.int64), np.zeros(S, np.int64), np.zeros(S, bool)
    p._si = SimpleNamespace(_args=lambda: (None, None, None, None))
    return p


@pytest.mark.parametrize("cfg", [(512, 128, True), (512, 128, False), (1024, 256, True), (512, 100, True)])
def test_inverse_plan_matches_inverse_pool(cfg, monkeypatch):
    n_fft, hop, center = cfg
    S, t = 10, 6
    rec = []
    monkeypatch.setattr(_C, "istft_pool_forward", lambda pool, lanes, X, A, n_max, T_max, *a: rec.append(lanes) or
                        torch.zeros(A, n_max))
    host = _host_inverse_pool(S, n_fft, hop, center)
    counters = np.zeros((3, S), np.int64)
    errors, info = np.zeros(S, np.int32), np.zeros((S, 2), np.int64)
    sticky = np.zeros(S, np.int32)
    rng = np.random.default_rng(n_fft + hop + center)
    X = torch.zeros(S, host.f_in, t, 2)
    seen = set()
    for step in range(150):
        restart = (rng.random(S) < 0.05) | (host.ended & (rng.random(S) < 0.3))
        if restart.any():
            host.reset(np.flatnonzero(restart))
            counters[:, restart] = 0
            errors[restart], info[restart], sticky[restart] = 0, 0, 0
        counts_in = rng.integers(0, t + 1, S) * (rng.random(S) < 0.7)
        counts_in = np.where(rng.random(S) < 0.03, t + 1, counts_in)
        end = rng.random(S) < 0.1
        length = np.where(rng.random(S) < 0.5, rng.integers(0, n_fft * 4, S), -1)

        def host_push(pool, c, e, ln):
            rows = np.flatnonzero(c)
            return pool.push(X[:len(rows)], rows, c[rows], e, ln)

        expect = np.zeros(S, np.int32)
        excs = {}
        for s in range(S):
            c, e = np.zeros(S, np.int64), np.zeros(S, bool)
            c[s], e[s] = counts_in[s], end[s]
            exc = _raises(lambda: host_push(copy.deepcopy(host), c, e, length))
            if exc is not None:
                excs[s] = exc
                msg = str(exc)
                expect[s] = (_C.LANE_ELENGTH if "counts must be" in msg else _C.LANE_EENDED if "has ended" in msg
                             else _C.LANE_ENOFRAMES if "without frames" in msg else _C.LANE_ELENGTH_SHORT)
        ok = expect == 0
        rec.clear()
        out = host_push(host, np.where(ok, counts_in, 0), end & ok, length)
        lanes, counts = _C.debug_device_istft_plan(counters, counts_in.astype(np.int32), end, length, errors, info, t,
                                                   n_fft, hop, center)
        want = np.zeros((S, 7), np.int64)
        want[:, 0], want[:, 1], want[:, 6] = np.arange(S), -1, -1
        want_counts = np.zeros(S, np.int64)
        if rec and len(rec[0]):
            h = rec[0].copy()
            h[:, 1] = np.where(h[:, 1] >= 0, h[:, 0], -1)  # the device pool's row s is slot s
            want[h[:, 0]] = h
        want_counts[out.slots.numpy()] = out.counts.numpy()
        assert (lanes == want).all(), (step, lanes, want)
        assert (counts == want_counts).all(), step
        assert (counters[0] == host.frames).all() and (counters[1] == host.emitted).all()
        assert (counters[2] == host.ended).all()
        fresh = sticky == 0
        sticky = np.where(sticky != 0, sticky, expect)
        assert (errors == sticky).all(), (step, errors, sticky)
        for s, e in excs.items():
            if not fresh[s] or expect[s] in seen:
                continue
            seen.add(expect[s])
            only = np.zeros(S, np.int32)
            only[s] = errors[s]
            view = _device_view(DeviceInversePool, S, only, info, frames_cap=t)
            with pytest.raises(type(e)) as got:
                view.check()
            assert str(got.value) == str(e), (got.value, e)
    assert seen >= {_C.LANE_ELENGTH, _C.LANE_EENDED, _C.LANE_ENOFRAMES}, seen


def _end_frames(total, K, hop, pad):
    return np.where(total + 2 * pad - K < 0, 0, (total + 2 * pad - K) // hop + 1)


def _ready(total, K, hop, pad, reflect):
    """``_ready_frames`` over an array."""
    need = K - pad
    f = np.where(total < need, 0, (total - need) // hop + 1)
    return np.where(reflect & (total < pad + 1), 0, f)


@pytest.mark.parametrize("K,hop", [(512, 128), (512, 256), (1024, 256), (400, 100), (255, 64), (2048, 512),
                                   (8760, 128), (1023, 37)])
@pytest.mark.parametrize("center,reflect", [(True, True), (True, False), (False, True)])
@pytest.mark.parametrize("chunk", [1, 100, 480, 1500])
def test_frame_cap_is_the_brute_force_maximum(K, hop, center, reflect, chunk):
    pad = K // 2 if center else 0
    refl = reflect and pad > 0
    assert all(_ready(np.array([v]), K, hop, pad, refl)[0] == _ready_frames(v, K, hop, pad, refl)
               for v in range(0, K + 3 * hop, 7))
    R = np.arange(0, K + 3 * hop + chunk)[:, None]  # past K + hop the counts repeat with period hop
    n = np.arange(0, chunk + 1)[None, :]
    r0, total = _ready(R, K, hop, pad, refl), R + n
    best = (_ready(total, K, hop, pad, refl) - r0).max()
    valid = (_end_frames(total, K, hop, pad) > 0) & ~(refl & (total <= pad))
    best = max(best, np.where(valid, _end_frames(total, K, hop, pad) - r0, 0).max())
    mode = _C.PAD_REFLECT if reflect else _C.PAD_CONSTANT
    assert _C.pool_frame_cap(chunk, K, hop, pad, mode) == best


@pytest.mark.parametrize("n_fft,hop", [(512, 128), (512, 256), (1024, 256), (512, 100), (256, 256), (400, 160)])
@pytest.mark.parametrize("center", [True, False])
@pytest.mark.parametrize("frames", [1, 3, 9])
def test_sample_cap_is_the_brute_force_maximum(n_fft, hop, center, frames):
    p = _host_inverse_pool(1, n_fft, hop, center)
    best = 0
    for F0 in range(0, n_fft // hop + 5):
        start = int(p._emit_end(np.array([F0]))[0])
        for T in range(0, frames + 1):
            n = F0 + T
            best = max(best, int(p._emit_end(np.array([n]))[0]) - start)
            if n > 0:
                for length in (-1, 10 ** 6):
                    best = max(best, int(p._flush_end(np.array([n]), np.array([length]))[0]) - start)
    assert _C.istft_pool_sample_cap(frames, n_fft, hop, center) == best


def test_construction_refusals_before_any_device_work():
    mfcc = features.MFCC(sr=16000, n_mfcc=20, n_fft=512, hop_length=128, verbose=False)
    with pytest.raises(ValueError, match="top_db"):
        DeviceStreamPool(mfcc, 4, 480)
    with pytest.raises(TypeError, match="StreamingPyramid"):
        DeviceStreamPool(features.CQT2010v2(sr=16000, n_bins=24, verbose=False), 4, 480)
    stft = features.STFT(n_fft=512, hop_length=128, verbose=False)
    with pytest.raises(ValueError):
        DeviceStreamPool(stft, 0, 480)
    with pytest.raises(ValueError):
        DeviceStreamPool(stft, 4, 0)
    with pytest.raises(ValueError):
        DeviceStreamPool(stft, 4, 480, dtype=torch.float64)
    with pytest.raises(TypeError):
        DeviceInversePool(stft, 4, 8)  # an STFT without iSTFT=True
    with pytest.raises(ValueError):
        DeviceInversePool(features.iSTFT(n_fft=512, hop_length=128, verbose=False), 4, 0)


def test_push_argument_checks_run_on_the_host():
    pool = DeviceStreamPool.__new__(DeviceStreamPool)
    pool.slots, pool.chunk, pool.dtype = 4, 300, torch.float32
    pool.ring = torch.zeros(4, 512)
    pool.counters = torch.zeros(3, 4, dtype=torch.int64)
    x, ln = torch.zeros(4, 300), torch.zeros(4, dtype=torch.int32)
    with pytest.raises(TypeError):
        pool.push(x.numpy(), ln)
    with pytest.raises(NotImplementedError):
        pool.push(x.requires_grad_(), ln)
    with pytest.raises(ValueError):
        pool.push(torch.zeros(4, 200), ln)
    with pytest.raises(ValueError):
        pool.push(torch.zeros(4, 300, dtype=torch.bfloat16), ln)
    with pytest.raises(TypeError):
        pool.push(torch.zeros(4, 300), [0, 0, 0, 0])
    with pytest.raises(TypeError):
        pool.push(torch.zeros(4, 300), ln.long())
    with pytest.raises(ValueError):
        pool.push(torch.zeros(4, 300), ln[:3])
    with pytest.raises(TypeError):
        pool.push(torch.zeros(4, 300), ln, torch.zeros(4, dtype=torch.int32))
    with pytest.raises(TypeError):
        pool.reset(torch.zeros(4, dtype=torch.int64))
