"""GPU: PyramidPool on seeded ragged schedules (idle slots, zero-length pushes, ends and restarts in the same slot,
NaN in every chunk column a slot does not take) against the whole-clip call on each stream, a one-stream
StreamingPyramid on the same packets (both bit for bit) and the fp64 oracle; 16-bit chunks, no synchronisation,
a launch count independent of the mix of clients, the SIMT path, and a cfg4-sized trace."""
import numpy as np
import pytest
import torch

from helpers import rel_errors, run_oracle
from nnaudio_b200 import _C
from nnaudio_b200.streaming import PyramidPool, StreamingPyramid
from test_zz_gpu_streaming_pyramid import CASES, _v2, _vqt

pytestmark = pytest.mark.gpu


def _run(pool, streams, seed, max_n, dtype=torch.float32, p_idle=0.2, p_end=0.5):
    """Feed each slot's streams (consumed in order) through `pool` in ragged pushes; returns, per slot, a list of
    (stream, its concatenated frames, its packet sizes)."""
    rng = np.random.default_rng(seed)
    S = pool.slots
    queue = [list(v) for v in streams]
    pos, parts, sizes = [0] * S, [[] for _ in range(S)], [[] for _ in range(S)]
    done = [[] for _ in range(S)]
    while any(queue):
        n = int(rng.integers(0, max_n))
        chunk = torch.full((S, n), float("nan"), device="cuda", dtype=dtype)
        lengths = np.zeros(S, np.int64)
        end = np.zeros(S, bool)
        for s in range(S):
            if not queue[s] or rng.random() < p_idle:
                continue
            x = queue[s][0]
            m = min(int(rng.integers(0, n + 1)), len(x) - pos[s])
            chunk[s, :m] = x[pos[s]:pos[s] + m]
            lengths[s] = m
            sizes[s].append(m)
            pos[s] += m
            end[s] = pos[s] == len(x) and rng.random() < p_end
        out = pool.push(chunk, lengths, end)
        for i, (s, c) in enumerate(zip(out.slots.tolist(), out.counts.tolist())):
            parts[s].append(out.frames[i:i + 1, :, :c])
            assert not out.frames[i, :, c:].any()  # exact zeros past the count
        for s in np.flatnonzero(end).tolist():
            done[s].append((queue[s].pop(0), torch.cat(parts[s], 2), sizes[s]))
            parts[s], sizes[s], pos[s] = [], [], 0
        pool.reset(np.flatnonzero(end))
    return done


def _one_stream(m, x, sizes, **kw):
    st = StreamingPyramid(m, 1, **kw)
    parts, pos = [], 0
    for n in sizes:
        parts.append(st.push(x[None, pos:pos + n]))
        pos += n
    parts.append(st.flush())
    return torch.cat(parts, 2)


@pytest.mark.parametrize("name", sorted(CASES))
def test_slots_equal_whole_clip_and_one_stream(name):
    cls, make, kw = CASES[name]
    m = make().cuda()
    g = torch.Generator(device="cuda").manual_seed(len(name))
    lens = [[30000, 25000], [40000], [26000, 27000], [33000], [45000], [28000, 29000]]
    streams = [[torch.randn(L, device="cuda", generator=g) for L in ls] for ls in lens]
    pool = PyramidPool(m, 6, **kw)
    done = _run(pool, streams, seed=len(name), max_n=6000)
    for s in range(6):
        assert len(done[s]) == len(streams[s])
        for x, y, sizes in done[s]:
            ref = m(x[None], **kw)
            assert y.shape == ref.shape, (name, s, y.shape, ref.shape)
            assert torch.equal(y, ref), (name, s, (y - ref).abs().max().item())
            assert torch.equal(y, _one_stream(m, x, sizes, **kw)), (name, s)


@pytest.mark.parametrize("name", ["v2_gen2", "v2_early"])
def test_oracle(name):
    cls, make, kw = CASES[name]
    m = make().cuda()
    g = torch.Generator(device="cuda").manual_seed(9)
    streams = [[torch.randn(30000, device="cuda", generator=g)] for _ in range(3)]
    done = _run(PyramidPool(m, 3, **kw), streams, seed=2, max_n=4000, p_end=1.0)
    for s in range(3):
        x, y, _ = done[s][0]
        want = run_oracle(cls, m, x[None].cpu().numpy(), kw)
        assert rel_errors(y.cpu().numpy(), want)[0] < 1e-4, (name, s)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("name", ["v2_gen2", "v2_early", "vqt_hop128"])
def test_half_chunks_equal_upcast(name, dtype):
    cls, make, kw = CASES[name]
    m = make().cuda()
    g = torch.Generator(device="cuda").manual_seed(4)
    streams = [[torch.randn(30000, device="cuda", generator=g).to(dtype)] for _ in range(4)]
    done = _run(PyramidPool(m, 4, **kw), streams, seed=3, max_n=5000, dtype=dtype, p_end=1.0)
    for s in range(4):
        x, y, _ = done[s][0]
        assert torch.equal(y, m(x[None].float(), **kw)), (name, s)


def test_steady_pushes_do_not_synchronise():
    m = _v2()().cuda()
    pool = PyramidPool(m, 8)
    x = torch.randn(8, 22050, device="cuda")
    lengths = np.array([2205, 0, 1000, 2205, 17, 2205, 300, 2205])
    for i in range(3):  # warm-up: packed operands
        pool.push(x[:, i * 2205:(i + 1) * 2205], lengths)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(3, 9):
            pool.push(x[:, i * 2205:(i + 1) * 2205], np.roll(lengths, i))
    finally:
        torch.cuda.set_sync_debug_mode("default")


@pytest.mark.parametrize("name", ["v2_gen2", "v2_early"])
def test_launch_count_does_not_depend_on_the_mix(name):
    _, make, kw = CASES[name]
    m = make().cuda()
    x = torch.randn(16, 200000, device="cuda")

    def launches(lengths):
        pool = PyramidPool(m, 16, **kw)
        pool.push(x[:, :100000], np.full(16, 100000))  # every stage and octave advances on the next push
        torch.cuda.synchronize()
        before = _C.launch_count()
        pool.push(x[:, 100000:], lengths)
        return _C.launch_count() - before

    full = launches(np.full(16, 100000))
    few = launches(np.array([100000, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 4096]))
    ragged = launches(np.arange(16) * 6000 + 4096)
    assert full == few == ragged


def test_simt_path_raises_and_keeps_state(monkeypatch):
    m = _vqt()().cuda()
    x = torch.randn(3, 40000, device="cuda")
    pool = PyramidPool(m, 3)
    pool.push(x[:, :20000], [20000, 15000, 0])
    before = (pool.received.copy(), pool.frames.copy(), pool.ended.copy(), pool.ring.clone())
    monkeypatch.setenv("NNAUDIO_B200_PATH", "simt")
    with pytest.raises(RuntimeError, match="no streamed tensor-core"):
        pool.push(x[:, 20000:], [20000, 20000, 5000], [True, False, False])
    assert np.array_equal(pool.received, before[0]) and np.array_equal(pool.frames, before[1])
    assert np.array_equal(pool.ended, before[2]) and torch.equal(pool.ring, before[3])
    monkeypatch.setenv("NNAUDIO_B200_PATH", "auto")
    out = pool.push(x[:, 20000:], [20000, 0, 0], [True, False, False])
    first = torch.cat([o for o in _slot_rows(out, 0)], 2)
    assert first.shape[2] > 0


def _slot_rows(out, s):
    return [out.frames[i:i + 1, :, :c] for i, (t, c) in enumerate(zip(out.slots.tolist(), out.counts.tolist()))
            if t == s]


def test_cfg4_trace():
    """cfg4 (CQT2010v2, 88 bins, 22.05 kHz, hop 512): 64 slots, streams of up to 30 s in 10-40 ms packets, idle
    slots, every ended stream bit for bit the whole-clip call."""
    m = _v2()().cuda()
    S, sr = 64, 22050
    rng = np.random.default_rng(12)
    g = torch.Generator(device="cuda").manual_seed(12)
    L = rng.integers(sr * 2, sr * 30, size=S)
    xs = [torch.randn(int(n), device="cuda", generator=g) for n in L]
    pool = PyramidPool(m, S)
    pos = np.zeros(S, np.int64)
    parts = [[] for _ in range(S)]
    checked = 0
    while (pos < L).any():
        n = int(rng.integers(sr // 100, sr * 4 // 100))
        take = np.where(rng.random(S) < 0.15, 0, np.minimum(n, L - pos))
        end = (pos + take == L) & (take > 0)
        chunk = torch.full((S, n), float("nan"), device="cuda")
        for s in np.flatnonzero(take).tolist():
            chunk[s, :take[s]] = xs[s][pos[s]:pos[s] + take[s]]
        out = pool.push(chunk, take, end)
        for i, (s, c) in enumerate(zip(out.slots.tolist(), out.counts.tolist())):
            parts[s].append(out.frames[i:i + 1, :, :c])
        pos += take
        for s in np.flatnonzero(end).tolist():
            assert torch.equal(torch.cat(parts[s], 2), m(xs[s][None])), s
            checked += 1
    assert checked == S
