"""Host logic of PyramidPool (no GPU): ragged schedules with idle slots, ends and restarts against the whole clip
on a float64 stand-in of the pool call, the vectorised counts against StreamingPyramid's scalar ones, the error
rules, the C entry point's host checks and its per-lane plan against the one-stream plan."""
import ctypes

import numpy as np
import pytest
import torch

from nnaudio_b200 import _C, features
from nnaudio_b200.streaming import PyramidPool, StreamingPyramid, StreamPool, StreamingTransform
from test_streaming_pyramid_host import CONFIGS, REPLAY, _install as _install_stream, _octaves64

import cpu_kernels


def _install(monkeypatch):
    """The pool call on float64 per-slot shadows: each lane's frames from its whole stream so far."""
    _install_stream(monkeypatch)
    shadow = {}

    def pool_forward(pool, lanes, x, A, T_max, **kw):
        bufs = shadow.setdefault(id(pool.ring), {})
        fmt = kw["out_format"]
        out = torch.zeros((A, kw["n_bins"], T_max) if fmt == _C.FMT_MAGNITUDE else (A, kw["n_bins"], T_max, 2))
        for i, (s, received, _, frames, n, end) in enumerate(lanes.tolist()):
            if received == 0:
                bufs[s] = torch.zeros(1, 0)
            if n > 0:
                bufs[s] = torch.cat([bufs[s], x[s:s + 1, :n].float()], 1)
            if i < A:  # frames past the lane's count are never read
                outs = _octaves64(bufs[s], kw)
                k = min(T_max, min(o.shape[2] for o in outs) - frames)
                c = torch.cat([o[:, :, frames:frames + k] for o in outs], 1)[:, -kw["n_bins"]:]
                y = cpu_kernels._format(cpu_kernels._scaled(c, kw["scale"], kw["scale_all"]), fmt, kw["sqrt_eps"])
                out[i, :, :k] = y[0]
        return out

    monkeypatch.setattr(_C, "cqt_pyramid_pool_forward", pool_forward)


def _schedule(pool, streams, seed, max_n=500):
    """Feed `streams` (list per slot of 1-D tensors, consumed in order) through `pool` in ragged pushes with idle
    slots, zero-length pushes and ends; returns per stream the concatenated frames."""
    rng = np.random.default_rng(seed)
    S = pool.slots
    queue = [list(v) for v in streams]
    pos = [0] * S
    parts = [[] for _ in range(S)]
    done = [[] for _ in range(S)]
    while any(queue):
        n = int(rng.integers(0, max_n))
        chunk = torch.full((S, n), float("nan"))
        lengths = np.zeros(S, np.int64)
        end = np.zeros(S, bool)
        for s in range(S):
            if not queue[s] or rng.random() < 0.2:
                continue
            x = queue[s][0]
            m = min(int(rng.integers(0, n + 1)), len(x) - pos[s])
            chunk[s, :m] = x[pos[s]:pos[s] + m]
            lengths[s] = m
            pos[s] += m
            end[s] = pos[s] == len(x) and rng.random() < 0.5
        out = pool.push(chunk, lengths, end)
        for i, (s, c) in enumerate(zip(out.slots.tolist(), out.counts.tolist())):
            parts[s].append(out.frames[i:i + 1, :, :c])
        for s in np.flatnonzero(end).tolist():
            done[s].append(torch.cat(parts[s], 2))
            parts[s] = []
            queue[s].pop(0)
            pos[s] = 0
        pool.reset(np.flatnonzero(end))
    return done


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_ragged_schedules_equal_whole_clip(name, monkeypatch):
    _install(monkeypatch)
    make, kw = CONFIGS[name]
    m = make()
    torch.manual_seed(3)
    streams = [[torch.randn(L) for L in lens] for lens in ([3000, 2500], [4100], [2600, 2700, 2800])]
    pool = PyramidPool(m, 3, **kw)
    done = _schedule(pool, streams, seed=len(name))
    for s, xs in enumerate(streams):
        assert len(done[s]) == len(xs)
        for x, y in zip(xs, done[s]):
            ref = m(x[None], **kw)
            assert y.shape == ref.shape, (name, s)
            assert torch.allclose(y, ref, rtol=1e-6, atol=1e-6), (name, s)


@pytest.mark.parametrize("name", ["vqt_reflect", "cqt2010v2_gen2"])
def test_vectorised_counts_equal_scalar(name, monkeypatch):
    _install(monkeypatch)
    m = CONFIGS[name][0]()
    pool, st = PyramidPool(m, 1), StreamingPyramid(m, 1)
    raw = np.arange(0, 6000, 13, dtype=np.int64)
    ready = pool._ready(raw)
    assert ready.tolist() == [st._ready(int(r)) for r in raw]
    assert pool._n_carry(raw, ready).tolist() == [st._n_carry(int(r), st._ready(int(r))) for r in raw]
    flushed = pool._counts(raw, np.ones(len(raw), bool))  # at an end every level has its whole-clip length
    for j, r in enumerate(raw.tolist()):
        want = [r]
        for _ in range(len(flushed) - 1):
            want.append(0 if want[-1] < 2 else (want[-1] - 2) // 2 + 1)
        assert [int(f[j]) for f in flushed] == want


def _raises(m, L):
    try:
        m(torch.randn(1, L))
    except RuntimeError:
        return True
    return False


def test_rules(monkeypatch):
    _install(monkeypatch)
    m = CONFIGS["vqt_reflect"][0]()
    with pytest.raises(ValueError):
        PyramidPool(m, 0)
    with pytest.raises(TypeError):
        PyramidPool(features.STFT(n_fft=64, hop_length=16, verbose=False), 2)
    with pytest.raises(TypeError, match="StreamingPyramid"):
        StreamPool(m, 2)
    with pytest.raises(TypeError):
        StreamingTransform(m, 2)
    pool = PyramidPool(m, 3)
    state = lambda: (pool.received.copy(), pool.frames.copy(), pool.ended.copy(), pool.dtype)  # noqa: E731

    def unchanged(fn, exc, match=None):
        before = state()
        with pytest.raises(exc, match=match):
            fn()
        after = state()
        assert all(np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b for a, b in zip(before, after))

    x = torch.zeros(3, 400)
    short = next(L for L in range(1, 400) if _raises(m, L))  # a length module(x) refuses
    unchanged(lambda: pool.push(x, [1, 2], None), ValueError)
    unchanged(lambda: pool.push(x, [1, 2, 500]), ValueError, "chunk width")
    unchanged(lambda: pool.push(x, [1.0, 2.0, 3.0]), TypeError)
    unchanged(lambda: pool.push(torch.zeros(3, 4, requires_grad=True), [1, 1, 1]), NotImplementedError)
    unchanged(lambda: pool.push(x, [400, short, 0], [False, True, False]), RuntimeError, "slot 1")
    pool.push(x, [400, 400, 0], [False, False, False])
    unchanged(lambda: pool.push(x.half(), [1, 1, 1]), ValueError, "dtype")
    pool.push(torch.randn(3, 3000), [3000, 3000, 0], [True, False, False])
    unchanged(lambda: pool.push(x, [1, 0, 0]), RuntimeError, "reset")
    unchanged(lambda: pool.push(x, [0, 0, 0], [True, False, False]), RuntimeError, "reset")
    pool.reset([0])
    pool.push(x, [1, 0, 0])
    pool.reset()
    assert pool.dtype is None and not pool.received.any()


def _grab():
    """A stand-in pool call that keeps the lane table PyramidPool.push builds."""
    captured = {}

    def grab(_, lanes, x, A, T_max, **kw):
        captured.update(lanes=lanes.copy(), A=A, T_max=T_max)
        return torch.zeros(A, kw["n_bins"], T_max)

    return grab, captured


def _call(lanes, A, T_max, slots, n, widths, hop, pad_mode, early=1):
    """nnab_cqt_pyramid_pool_forward's host checks (dummy device pointers: an EINVAL returns before any use)."""
    L = _C.lib()
    a = np.ascontiguousarray(np.asarray(lanes, np.int64).reshape(-1, 6))
    p = ctypes.c_void_p(256)
    n_oct = len(widths)
    arr = (ctypes.c_void_p * n_oct)(*([256] * n_oct))
    return L.nnab_cqt_pyramid_pool_forward(
        p, a.ctypes.data_as(ctypes.c_void_p) if len(a) else None, p, len(a), A, p, _C.DTYPE_F32, slots, n, n, n_oct,
        arr, arr, arr, (ctypes.c_int32 * n_oct)(*widths), 12, p, p, p if early > 1 else None, p if early > 1 else None,
        early, hop, pad_mode, 12 * n_oct, None, 1.0, _C.FMT_MAGNITUDE, 0.0, p, T_max, None, 0, 0, None)


def test_c_entry_host_checks(monkeypatch):
    _install(monkeypatch)
    m = CONFIGS["vqt_reflect"][0]()
    pool = PyramidPool(m, 4)
    grab, cap = _grab()
    monkeypatch.setattr(_C, "cqt_pyramid_pool_forward", grab)
    pool.push(torch.zeros(4, 3000), [3000, 2000, 2500, 0])
    pool.push(torch.zeros(4, 700), [700, 300, 0, 650], [True, False, False, False])
    lanes, A, T_max = cap["lanes"], cap["A"], cap["T_max"]
    widths, hop, pm = pool.widths, pool.hop, _C.PAD_REFLECT
    EINVAL = -1
    assert A >= 1 and len(lanes) == 3
    ws = _C.cqt_pyramid_pool_workspace_bytes(lanes, A, T_max, widths, hop, 1, pm)  # host-only
    assert ws > 0
    assert _C.cqt_pyramid_pool_workspace_bytes(lanes, A, T_max + 1, widths, hop, 1, pm) == 0
    bad_order = lanes[::-1].copy() if A == len(lanes) else np.concatenate([lanes[A:], lanes[:A]])
    assert _call(bad_order, A, T_max, 4, 700, widths, hop, pm) == EINVAL
    rep = lanes.copy()
    rep[1, 0] = rep[0, 0]
    assert _call(rep, A, T_max, 4, 700, widths, hop, pm) == EINVAL
    imp = lanes.copy()
    imp[0, 2] += 1  # n_carry no stream has
    assert _call(imp, A, T_max, 4, 700, widths, hop, pm) == EINVAL
    assert _call(lanes, A + 1 if A < len(lanes) else A - 1, T_max, 4, 700, widths, hop, pm) == EINVAL
    assert _call(lanes, A, T_max + 1, 4, 700, widths, hop, pm) == EINVAL
    assert _call(lanes, A, T_max, 4, 100, widths, hop, pm) == EINVAL  # a lane n above the chunk width
    short = np.array([[0, 0, 0, 0, 10, 1]], np.int64)  # an end on a stream far too short
    assert _call(short, 0, 0, 4, 10, widths, hop, pm) == EINVAL


@pytest.mark.parametrize("name", sorted(REPLAY))
def test_pool_plan_equals_one_stream_plan(name, monkeypatch):
    _install(monkeypatch)
    m = REPLAY[name]()
    pool = PyramidPool(m, 5)
    grab, cap = _grab()
    monkeypatch.setattr(_C, "cqt_pyramid_pool_forward", grab)
    rng = np.random.default_rng(5)
    widths, hop, early, pm = pool.widths, pool.hop, pool.early, _C.PAD_REFLECT
    checked = 0
    for step in range(40):
        n = int(rng.integers(0, 1500))
        lengths = np.where(rng.random(5) < 0.3, 0, rng.integers(0, n + 1, 5))
        end = (pool.received + lengths > 12000) & (rng.random(5) < 0.5)
        if not ((lengths > 0) | end).any():
            continue
        pool.push(torch.zeros(5, n), lengths, end)
        lanes, A = cap["lanes"], cap["A"]
        plans = _C.cqt_pyramid_pool_plan(lanes, A, widths, hop, pm, early)
        for (s, rec, nc, frm, nn, e), got in zip(lanes.tolist(), plans):
            assert got == _C.cqt_pyramid_chunk_plan(rec, nc, frm, nn, e, widths, hop, pm, early)
            checked += 1
        pool.reset(np.flatnonzero(end))
    assert checked > 40


@pytest.mark.parametrize("name", sorted(REPLAY))
def test_lock_step_workspace_equals_pool_of_its_lanes(name, monkeypatch):
    """A StreamingPyramid push of B streams is a pool push of B lanes with its counters in slots 0 .. B-1: over
    seeded push sequences ending in a flush, the chunk call's workspace query equals the pool's for that table."""
    _install(monkeypatch)
    st = StreamingPyramid(REPLAY[name](), 1)
    widths, hop, early, pm = st.widths, st.hop, st.early, _C.PAD_REFLECT
    w = (ctypes.c_int32 * len(widths))(*widths)
    rng = np.random.default_rng(9)
    for B in (1, 3):
        received = n_carry = frames = 0
        for step in range(30):
            n, flush = int(rng.integers(1, 3000)), int(step == 29)
            _, t_end = _C.cqt_pyramid_chunk_plan(received, n_carry, frames, n, flush, widths, hop, pm, early)
            T = t_end - frames
            lanes = [[b, received, n_carry, frames, n, flush] for b in range(B)]
            want = _C.cqt_pyramid_pool_workspace_bytes(lanes, B if T > 0 else 0, T, widths, hop, early, pm)
            got = _C.lib().nnab_cqt_pyramid_chunk_workspace_bytes(B, received, n_carry, frames, n, flush,
                                                                   len(widths), w, hop, early, pm)
            assert want > 0 and got == want, (name, B, step)
            received += n
            frames = t_end
            n_carry = st._n_carry(received, frames)
