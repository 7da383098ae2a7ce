"""CPU: the host logic of nnaudio_b200.streaming.StreamPool against whole-clip float64 stand-ins for the C calls.

As in tests/test_streaming_host.py, two stand-ins replace the ``_C.*_pool_forward`` calls: "fused" returns the
frames the library must return (row i: the float64 transform of lane i's stream so far, its new frames, zeros
up to T_max); "concat" reports NNAB_EUNSUPPORTED, so the pool's own concat route (one index gather per push,
the mask, the carry ring) runs on the offline stand-in.  Seeded ragged schedules with ends and restarts must
give every stream its whole-clip frames.  The C entry points' host checks are called with fake pointers.
"""
import ctypes

import numpy as np
import pytest
import torch

import cpu_kernels
from nnaudio_b200 import _C
from nnaudio_b200.streaming import StreamingTransform, StreamPool, _ready_frames
from test_streaming_host import _OFFLINE64, CONFIGS


def _pool_standin(name, calls):
    offline = _OFFLINE64[name]
    shadow = {}

    def pool_forward(pool, lanes, x, A, T_max, **kw):
        calls.append(A)
        rows = []
        for i, (s, R, _, F0, n, end) in enumerate(lanes.tolist()):
            buf = shadow.setdefault((id(pool), s), [])
            if R == 0:
                buf.clear()
            if n > 0:
                buf.append(x[s:s + 1, :n].double())
            if i >= A:
                continue
            full = offline(torch.cat(buf, 1), **kw)
            T = (full.shape[2] if end else _ready_frames(R + n, pool.K, pool.hop, pool.pad, pool._reflect)) - F0
            row = torch.zeros((1,) + full.shape[1:2] + (T_max,) + full.shape[3:], dtype=full.dtype)
            row[:, :, :T] = full[:, :, F0:F0 + T]
            rows.append(row)
        return torch.cat(rows, 0) if rows else pool._st._empty(name, kw)[:0]

    return pool_forward


def _install(monkeypatch, mode):
    cpu_kernels.install(monkeypatch)
    calls = []
    for name in _OFFLINE64:
        monkeypatch.setattr(_C, name, _OFFLINE64[name])
        fn = _pool_standin(name, calls) if mode == "fused" else (lambda *a, **k: None)
        monkeypatch.setattr(_C, name.replace("_forward", "_pool_forward"), fn)
    return calls


def _schedule(S, K, hop, seed, steps=60):
    """(lengths, end, reset-before) per push: ragged, zero-length and one-sample packets, one slot taking a long
    packet while the others take one sample, slots ending mid-run and reset a few pushes later."""
    rng = np.random.default_rng(seed)
    ended = np.zeros(S, bool)
    since_end = np.zeros(S, int)
    total = np.zeros(S, int)
    out = []
    for step in range(steps):
        reset = np.flatnonzero(ended & (since_end >= 2) & (rng.random(S) < 0.5))
        ended[reset] = False
        total[reset] = 0
        kind = step % 6
        if kind == 0:
            lengths = rng.integers(0, 3 * hop, size=S)
        elif kind == 1:
            lengths = np.ones(S, int)
            lengths[rng.integers(S)] = 5 * K + 7
        elif kind == 2:
            lengths = rng.choice([0, 1, hop - 1, hop, K // 2 + 1], size=S)
        else:
            lengths = rng.integers(0, 2 * K, size=S)
        lengths[ended] = 0
        total += lengths
        end = ~ended & (total >= K + hop) & (rng.random(S) < 0.08)
        ended |= end
        since_end = np.where(end, 0, since_end + 1)
        out.append((lengths, end, reset))
    lengths = np.zeros(S, int)
    end = ~ended & (total > K)  # the streams still open end in a last push (the too-short ones are dropped)
    out.append((lengths, end, np.zeros(0, int)))
    return out


@pytest.mark.parametrize("mode", ["fused", "concat"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_ragged_schedule_gives_every_stream_its_whole_clip(name, mode, monkeypatch):
    _install(monkeypatch, mode)
    make, kw = CONFIGS[name]
    m = make()
    S = 5 + len(name) % 4
    pool = StreamPool(m, S, **kw)
    gen = torch.Generator().manual_seed(len(name))
    live = [[] for _ in range(S)]   # samples and rows of the stream in each slot
    rows = [[] for _ in range(S)]
    done = []
    for lengths, end, reset in _schedule(S, pool.K, pool.hop, seed=len(name) * 7 + (mode == "fused")):
        if len(reset):
            pool.reset(reset.tolist())
            for s in reset:
                live[s], rows[s] = [], []
        n = int(lengths.max())
        chunk = torch.randn(S, n, generator=gen)
        before_frames, ended_before = pool.frames.copy(), pool.ended.copy()
        out = pool.push(chunk, lengths.tolist(), end.tolist())
        for s in range(S):
            live[s].append(chunk[s, :lengths[s]])
        want = []
        for s in range(S):
            total = int(pool.received[s])
            if ended_before[s]:
                T = before_frames[s]
            elif end[s]:
                T = (total + 2 * pool.pad - pool.K) // pool.hop + 1
            else:
                T = _ready_frames(total, pool.K, pool.hop, pool.pad, pool._reflect)
            assert pool.frames[s] == T, (s, pool.frames[s], T)
            if T > before_frames[s]:
                want.append((s, T - before_frames[s]))
        assert out.slots.tolist() == [s for s, _ in want], "ascending, exactly the slots with new frames"
        assert out.counts.tolist() == [c for _, c in want]
        assert out.frames.shape[0] == len(want)
        T_max = max([c for _, c in want], default=0)
        assert out.frames.shape[2] == T_max
        for i, (s, c) in enumerate(want):
            assert (out.frames[i, :, c:] == 0).all(), "padded frames are exact zeros"
            rows[s].append(out.frames[i:i + 1, :, :c])
        for s in np.flatnonzero(end):
            done.append((torch.cat(live[s]), torch.cat(rows[s], 2)))
    assert len(done) >= S
    for x, got in done:
        ref = m(x[None].double() if mode == "fused" else x[None], **kw)
        assert got.shape == ref.shape, (name, got.shape, ref.shape)
        d = (got - ref).double()
        if name == "stft_phase":  # float64 round-off may put an angle of pi on either side of the cut
            d = torch.remainder(d + np.pi, 2 * np.pi) - np.pi
        assert d.abs().max().item() <= 1e-12 * max(ref.abs().max().item(), 1e-30), (name, mode)


@pytest.mark.parametrize("mode", ["fused", "concat"])
def test_pool_streams_match_one_streaming_transform_each(mode, monkeypatch):
    """The same packets through a one-stream StreamingTransform give the same frames, push by push."""
    _install(monkeypatch, mode)
    import test_streaming_host as sh
    for name in sh._OFFLINE64:
        monkeypatch.setattr(_C, name.replace("_forward", "_chunk_forward"),
                            sh._fused_standin(name) if mode == "fused" else (lambda *a, **k: None))
    make, kw = CONFIGS["mel"]
    m = make()
    pool = StreamPool(m, 3)
    one = [StreamingTransform(m, 1) for _ in range(3)]
    rng = np.random.default_rng(5)
    x = torch.randn(3, 2000)
    pos = np.zeros(3, int)
    while (pos < 2000).any():
        lengths = np.minimum(rng.integers(0, 90, size=3), 2000 - pos)
        chunk = torch.zeros(3, int(lengths.max()))
        for s in range(3):
            chunk[s, :lengths[s]] = x[s, pos[s]:pos[s] + lengths[s]]
        out = pool.push(chunk, lengths, (pos < 2000) & (pos + lengths >= 2000))
        got = dict(zip(out.slots.tolist(), range(len(out.slots))))
        for s in range(3):
            piece = x[s:s + 1, pos[s]:pos[s] + lengths[s]]
            if pos[s] < 2000:
                ref = one[s].push(piece)
                if pos[s] + lengths[s] >= 2000:
                    ref = torch.cat([ref, one[s].flush()], 2)
            else:
                ref = torch.zeros(1, 12, 0)
            if ref.shape[2]:
                i = got[s]
                assert torch.allclose(out.frames[i:i + 1, :, :ref.shape[2]].double(), ref.double(), rtol=0,
                                      atol=1e-12 * ref.abs().max().item())
            else:
                assert s not in got
        pos += lengths


def test_rules_and_errors_change_nothing(monkeypatch):
    calls = _install(monkeypatch, "fused")
    make, kw = CONFIGS["stft_mag"]
    m = make()
    with pytest.raises(ValueError):
        StreamPool(m, _C.MAX_BATCH + 1)
    pool = StreamPool(m, 4)
    pool.push(torch.randn(4, 50), [50, 10, 0, 3])

    def state():
        return pool.received.copy(), pool.frames.copy(), pool.ended.copy(), len(calls)

    s0 = state()
    with pytest.raises(ValueError):
        pool.push(torch.randn(4, 10), [11, 0, 0, 0])  # lengths[s] > n
    with pytest.raises(ValueError):
        pool.push(torch.randn(4, 10, dtype=torch.bfloat16), [1, 1, 1, 1])  # dtype fixed by the first push
    with pytest.raises(ValueError):
        pool.push(torch.randn(4, 10), [1, 1, 1])  # one length per slot
    with pytest.raises(TypeError):
        pool.push(torch.randn(4, 10), [1.5, 1, 1, 1])
    with pytest.raises(NotImplementedError):
        pool.push(torch.randn(4, 10, requires_grad=True), [1, 1, 1, 1])
    # an end on a stream too short for the module: the exception module(x) raises, naming the slot; nothing
    # runs and no counter moves, for the other slots of the call either
    with pytest.raises(AssertionError, match="slot 1"):
        pool.push(torch.randn(4, 10), [10, 10, 0, 10], [True, True, False, False])
    with pytest.raises(RuntimeError, match="slot 3"):
        pool.push(torch.randn(4, 29), [0, 0, 0, 29], [False, False, False, True])  # reflect needs pad < L
    assert all(np.array_equal(a, b) for a, b in zip(state()[:3], s0[:3])) and state()[3] == s0[3]
    out = pool.push(torch.randn(4, 10), [10, 0, 0, 0], [True, False, False, False])
    assert out.slots.tolist() == [0] and out.counts.tolist() == [(60 + 64 - 64) // 16 + 1 - 2]
    with pytest.raises(RuntimeError, match="slot 0"):
        pool.push(torch.randn(4, 1), [1, 0, 0, 0])  # an ended slot takes nothing ...
    with pytest.raises(RuntimeError, match="slot 0"):
        pool.push(torch.randn(4, 0), [0, 0, 0, 0], [True, False, False, False])  # ... and no second end
    out = pool.push(torch.randn(4, 0), [0, 0, 0, 0])  # an empty push
    assert out.frames.shape[0] == 0 and out.slots.numel() == 0
    with pytest.raises(TypeError):
        pool.reset(np.array([0.0]))  # slots are integers, as in InversePool.reset
    assert pool.ended[0]
    pool.reset([0])
    assert pool.received[0] == 0 and not pool.ended[0] and pool.received[1] == 10
    assert pool.push(torch.randn(4, 100), [100, 0, 0, 0]).counts.tolist() == [_ready_frames(100, 64, 16, 32, True)]
    with pytest.raises(TypeError):
        pool.push(torch.randn(4, 1), torch.ones(4, dtype=torch.int64, device="meta"))  # lengths stay on the CPU


def test_strict_pool_refuses_the_concat_route(monkeypatch):
    _install(monkeypatch, "concat")
    make, kw = CONFIGS["mel"]
    pool = StreamPool(make(), 2, _strict=True)
    with pytest.raises(RuntimeError, match="no fused pool route"):
        pool.push(torch.randn(2, 200), [200, 100])
    # nothing ran, so nothing is committed: not the counters, not the sample type
    assert pool.dtype is None and not pool.received.any() and not pool.frames.any()
    with pytest.raises(RuntimeError, match="no fused pool route"):
        pool.push(torch.randn(2, 200, dtype=torch.bfloat16), [200, 100])


# ------------------------------------------------------------------------------------------- C host checks
EINVAL = -1


def _lanes(*rows):
    flat = [int(v) for r in rows for v in r]
    return (ctypes.c_int64 * max(len(flat), 1))(*flat)


def _entry_points():
    lib = _C.lib()
    P = ctypes.c_void_p
    ring = chunk = w = out = dl = P(256)  # never dereferenced on the host

    def stft(lanes, n_lanes, A, T_max, n):
        return lib.nnab_stft_pool_forward(ring, lanes, dl, n_lanes, A, chunk, 0, 4, n, n, w, w, None, 64, 33, 16,
                                          1, 0, 0, 0.0, out, T_max, None, 0, 0, None)

    def fbank(lanes, n_lanes, A, T_max, n):
        return lib.nnab_stft_filterbank_pool_forward(ring, lanes, dl, n_lanes, A, chunk, 0, 4, n, n, w, w, None, 64,
                                                     33, 16, 1, 0, 0.0, 2.0, w, 12, None, out, T_max, None, 0, 0,
                                                     None)

    def mfcc(lanes, n_lanes, A, T_max, n):
        return lib.nnab_mfcc_pool_forward(ring, lanes, dl, n_lanes, A, chunk, 0, 4, n, n, w, w, None, 64, 33, 16,
                                          1, 0, 0.0, 2.0, w, 12, None, 1e-10, 1.0, -1.0, w, 8, out, T_max, None, 0,
                                          0, None)

    def cqt(lanes, n_lanes, A, T_max, n):
        return lib.nnab_cqt1992v2_pool_forward(ring, lanes, dl, n_lanes, A, chunk, 0, 4, n, n, w, w, None, None,
                                               None, 24, 64, 16, 1, 0, None, 1.0, 0, 0.0, out, T_max, None, 0, 0,
                                               None)

    return {"stft": stft, "filterbank": fbank, "mfcc": mfcc, "cqt1992v2": cqt}


@pytest.mark.parametrize("entry", ["stft", "filterbank", "mfcc", "cqt1992v2"])
def test_pool_entry_points_reject_bad_lane_tables_on_the_host(entry):
    call = _entry_points()[entry]
    # K = 64, hop 16, reflect centre padding: after 100 samples a new stream has 5 ready frames, after 40 one
    fresh = lambda s, n=100, end=0: (s, 0, 0, 0, n, end)  # noqa: E731
    assert call(_lanes(fresh(0), fresh(2, 40)), 2, 2, 4, 100) == EINVAL, "T_max is the longest row's count"
    assert call(_lanes(fresh(0), fresh(2, 40)), 2, 1, 5, 100) == EINVAL, "A counts the lanes with frames"
    assert call(_lanes(fresh(2), fresh(0, 40)), 2, 2, 5, 100) == EINVAL, "slots ascend within a group"
    assert call(_lanes(fresh(0), fresh(0, 40)), 2, 2, 5, 100) == EINVAL, "a slot appears once"
    assert call(_lanes(fresh(1), fresh(1, 10)), 2, 1, 5, 100) == EINVAL, "a slot appears once across groups"
    assert call(_lanes(fresh(1, 10), fresh(2)), 2, 1, 5, 100) == EINVAL, "the lanes with frames come first"
    assert call(_lanes(fresh(4)), 1, 1, 5, 100) == EINVAL, "slot out of range"
    assert call(_lanes(fresh(0)), 1, 1, 5, 50) == EINVAL, "a lane's n is at most the chunk width"
    assert call(_lanes((0, 100, 10, 5, 0, 1)), 1, 1, 1, 0) == EINVAL, "counters no stream can have"
    assert call(_lanes((0, 100, 36, 4, 0, 0)), 1, 0, 0, 0) == EINVAL, "frames must be every ready frame"
    assert call(_lanes(fresh(0, 20, 1)), 1, 1, 1, 100) == EINVAL, "an end needs pad < the stream's length"
    assert call(_lanes(fresh(0, 0, 0)), 1, 0, 0, 100) == EINVAL, "a lane with nothing to do"
    assert call(_lanes(fresh(0, 100, 2)), 1, 1, 7, 100) == EINVAL, "end is 0 or 1"
    assert call(None, 1, 1, 5, 100) == EINVAL, "no host table"


def test_pool_workspace_queries_equal_the_offline_queries():
    lib = _C.lib()
    for path in (_C.PATH_AUTO, _C.PATH_SIMT):
        for A, T_max in ((1, 1), (3, 5), (256, 12)):
            L = 16 * (T_max - 1) + 64
            assert lib.nnab_stft_pool_workspace_bytes(A, T_max, 64, 33, 16, path) == \
                lib.nnab_stft_workspace_bytes(A, L, 64, 33, 16, 0, path)
            assert lib.nnab_filterbank_pool_workspace_bytes(A, T_max, 64, 33, 16, 12, path, 1) == \
                lib.nnab_filterbank_workspace_bytes(A, L, 64, 33, 16, 0, 12, path, 1)
            assert lib.nnab_mfcc_pool_workspace_bytes(A, T_max, 64, 33, 16, 12, path, 0) == \
                lib.nnab_mfcc_workspace_bytes(A, L, 64, 33, 16, 0, 12, path, 0)
            assert lib.nnab_cqt1992v2_pool_workspace_bytes(A, T_max, 64, 24, 16, path) == \
                lib.nnab_cqt1992v2_workspace_bytes(A, L, 64, 24, 16, 0, path)
    assert lib.nnab_stft_pool_workspace_bytes(0, 5, 64, 33, 16, 0) == 0
    assert lib.nnab_stft_pool_workspace_bytes(3, 0, 64, 33, 16, 0) == 0


@pytest.mark.parametrize("K, hop, center, pm", [(64, 16, 1, _C.PAD_REFLECT), (64, 16, 1, _C.PAD_CONSTANT),
                                                (400, 160, 0, _C.PAD_REFLECT), (512, 128, 1, _C.PAD_REFLECT)])
def test_lock_step_workspace_equals_pool_of_its_lanes(K, hop, center, pm):
    """A lock-step push of B streams is a pool push of B lanes that share its counters: over seeded push sequences
    ending in a flush, each chunk call's workspace query equals its pool query for A = B (0 when the push returns no
    frame) and T_max = the push's frames."""
    lib = _C.lib()
    pad, F = K // 2 if center else 0, K // 2 + 1
    rng = np.random.default_rng(K + hop + pm)
    for path in (_C.PATH_AUTO, _C.PATH_SIMT):
        for B in (1, 3, 256):
            received = frames = 0
            for step in range(25):
                n, flush = int(rng.choice([0, 1, hop, int(rng.integers(0, 3 * K))])), int(step == 24)
                total = received + n
                t_end = ((total + 2 * pad - K) // hop + 1 if flush
                         else _ready_frames(total, K, hop, pad, pm == _C.PAD_REFLECT))
                T = t_end - frames
                A, head = (B if T > 0 else 0), (B, received, frames, n, flush)
                assert lib.nnab_stft_chunk_workspace_bytes(*head, K, F, hop, center, pm, path) == \
                    lib.nnab_stft_pool_workspace_bytes(A, T, K, F, hop, path), (B, step)
                for has_table in (0, 1):
                    assert lib.nnab_filterbank_chunk_workspace_bytes(*head, K, F, hop, center, pm, 12, path,
                                                                     has_table) == \
                        lib.nnab_filterbank_pool_workspace_bytes(A, T, K, F, hop, 12, path, has_table), (B, step)
                    assert lib.nnab_mfcc_chunk_workspace_bytes(*head, K, F, hop, center, pm, 12, path, has_table) == \
                        lib.nnab_mfcc_pool_workspace_bytes(A, T, K, F, hop, 12, path, has_table), (B, step)
                assert lib.nnab_cqt1992v2_chunk_workspace_bytes(*head, K, 24, hop, center, pm, path) == \
                    lib.nnab_cqt1992v2_pool_workspace_bytes(A, T, K, 24, hop, path), (B, step)
                received, frames = total, t_end
            assert frames > 0
