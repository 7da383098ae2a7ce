"""GPU: DevicePyramidPool against PyramidPool on the same seeded serving traces, eagerly and as one CUDA graph
replayed tick by tick with its inputs updated in place.

Every tick, row s of the device pool (up to its count) must equal PyramidPool's row for slot s bit for bit, rows past
their counts must be exact zeros, the replayed graph must equal the eager pushes bit for bit, the eager pushes must not
synchronise, and completed streams must equal ``module(x)`` (16-bit streams: ``module(x.float())``).  The chunk
columns a slot does not take hold NaN.  Also: dropped slots and ``check()``, a launch count and an allocation state
that do not depend on the traffic, the SIMT path, a cfg4-sized trace, and one graph that runs a DeviceStreamPool Mel
front end and a DevicePyramidPool on the same packets.
"""
import numpy as np
import pytest
import torch

from nnaudio_b200 import _C, features
from nnaudio_b200.streaming import DevicePyramidPool, DeviceStreamPool, PyramidPool, StreamPool
from test_zz_gpu_streaming_pyramid import CASES, _v2

pytestmark = pytest.mark.gpu

NAMES = ["v2_gen2", "v2_gen2_complex", "v2_gen2_phase", "v2_constant", "v2_hop128", "v2_early", "cqt2010",
         "vqt_gamma5"]


def _trace(S, chunk, ticks, seed, min_end):
    """[(lengths, end, restart)] per tick: ragged packets, ~20 % idle slots, ends on streams long enough for the
    module, the ended slots restarted the next tick."""
    rng = np.random.default_rng(seed)
    total = np.zeros(S, int)
    ended = np.zeros(S, bool)
    out = []
    for _ in range(ticks):
        restart = ended.copy()
        total[restart] = 0
        ended[:] = False
        lengths = rng.integers(0, chunk + 1, size=S) * (rng.random(S) < 0.8)
        total += lengths
        end = (total > min_end) & (rng.random(S) < 0.1)
        ended |= end
        out.append((lengths, end, restart))
    return out


def _inputs(tr, S, chunk, dtype, seed):
    """Each tick's chunk, NaN in the columns a slot does not take."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    xs = torch.randn(len(tr), S, chunk, device="cuda", generator=gen).to(dtype)
    for i, (ln, _, _) in enumerate(tr):
        cols = torch.arange(chunk, device="cuda")[None] >= torch.as_tensor(ln, device="cuda")[:, None]
        xs[i][cols] = float("nan")
    return xs


def _graph(pool, S, chunk, dtype):
    """A CUDA graph of one tick (reset where `restart`, then the push) on in-place inputs."""
    x = torch.zeros(S, chunk, device="cuda", dtype=dtype)
    lengths = torch.zeros(S, dtype=torch.int32, device="cuda")
    end = torch.zeros(S, dtype=torch.bool, device="cuda")
    restart = torch.zeros(S, dtype=torch.bool, device="cuda")
    pool.reset(restart)
    pool.push(x, lengths, end)  # eager warm-up tick (every slot idle)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pool.reset(restart)
        pool.push(x, lengths, end)
    return g, (x, lengths, end, restart)


def _run(name, dtype, S=5, chunk=3000, ticks=70, seed=0):
    _, make, kw = CASES[name]
    m = make().cuda()
    host = PyramidPool(m, S, **kw)
    tr = _trace(S, chunk, ticks, seed, min_end=30000)
    xs = _inputs(tr, S, chunk, dtype, seed)
    eager = DevicePyramidPool(m, S, chunk, dtype, **kw)
    graphed = DevicePyramidPool(m, S, chunk, dtype, **kw)
    g, ins = _graph(graphed, S, chunk, dtype)
    streams, rows, done = [[] for _ in range(S)], [[] for _ in range(S)], []
    for i, (ln, en, rs) in enumerate(tr):
        dev_in = (torch.as_tensor(ln, dtype=torch.int32).cuda(), torch.as_tensor(en).cuda(), torch.as_tensor(rs).cuda())
        if rs.any():
            host.reset(np.flatnonzero(rs))
        out = host.push(xs[i], ln, en)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            eager.reset(dev_in[2])
            eager.push(xs[i], dev_in[0], dev_in[1])
        finally:
            torch.cuda.set_sync_debug_mode(0)
        for a, b in zip(ins, (xs[i],) + dev_in):
            a.copy_(b)
        g.replay()
        assert torch.equal(graphed.frames, eager.frames) and torch.equal(graphed.counts, eager.counts), (name, i)
        counts = eager.counts.cpu().numpy()
        want = np.zeros(S, int)
        want[out.slots.numpy()] = out.counts.numpy()
        assert (counts == want).all(), (name, i, counts, want)
        for r, s in enumerate(out.slots.tolist()):
            assert torch.equal(eager.frames[s, :, :counts[s]], out.frames[r, :, :counts[s]]), (name, i, s)
        tail = eager.frames.clone()
        for s in range(S):
            tail[s, :, :counts[s]] = 0
        assert torch.count_nonzero(tail).item() == 0, "frames past the counts are exact zeros"
        for s in range(S):
            if rs[s]:
                streams[s], rows[s] = [], []
            streams[s].append(xs[i, s, :ln[s]])
            rows[s].append(eager.frames[s:s + 1, :, :counts[s]].clone())
            if en[s]:
                done.append((torch.cat(streams[s]), torch.cat(rows[s], 2)))
    assert eager.errors.count_nonzero().item() == 0 and graphed.errors.count_nonzero().item() == 0
    return m, kw, done


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("name", NAMES)
def test_device_pool_equals_pyramid_pool_eager_and_graph(name, dtype):
    with torch.no_grad():
        m, kw, done = _run(name, dtype, seed=len(name))
        assert len(done) >= 3, len(done)
        for x, got in done[:3]:
            ref = m(x[None].float(), **kw)
            assert torch.equal(got, ref), (name, (got - ref).abs().max().item())


def test_float16_stream():
    with torch.no_grad():
        m, kw, done = _run("v2_gen2", torch.float16, seed=16)
        assert len(done) >= 3
        for x, got in done[:3]:
            assert torch.equal(got, m(x[None].float(), **kw))


def test_errors_drop_the_slot_and_check_raises_the_host_type():
    m = _v2()().cuda()
    S, chunk = 4, 2000
    pool = DevicePyramidPool(m, S, chunk)
    x = torch.randn(S, chunk, device="cuda")
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")  # noqa: E731
    b = lambda v: torch.tensor(v, dtype=torch.bool, device="cuda")  # noqa: E731
    with torch.no_grad():
        for _ in range(20):
            pool.push(x, i32([2000, 2000, 2000, 0]))
        pool.push(x, i32([2000, 2000, 2000, 0]), b([0, 0, 1, 0]))
        before = pool.counters.clone()
        ref = DevicePyramidPool(m, S, chunk)  # slot 0 alone, the same packets
        for _ in range(20):
            ref.push(x, i32([2000, 0, 0, 0]))
        ref.push(x, i32([2000, 0, 0, 0]))
        ref.push(x, i32([2000, 0, 0, 0]))
        pool.push(x, i32([2000, 2001, 100, 0]), b([0, 0, 0, 1]))  # slot 1: too long, 2: ended, 3: too short
        assert pool.errors.tolist() == [0, _C.LANE_ELENGTH, _C.LANE_EENDED, _C.LANE_ESHORT]
        assert torch.equal(pool.counters[:, 1:], before[:, 1:]), "dropped slots keep their counters"
        assert pool.counts[1:].count_nonzero().item() == 0 and pool.frames[1:].count_nonzero().item() == 0
        assert torch.equal(pool.frames[0], ref.frames[0]) and pool.counts[0] == ref.counts[0], "slot 0 is untouched"
        assert pool.counters[0, 0].item() == 22 * 2000
        with pytest.raises(ValueError, match="slot 1 has 2001"):
            pool.check()
        host = PyramidPool(m, S)
        with pytest.raises(ValueError, match="slot 1 has 2001"):
            host.push(x, [2000, 2001, 100, 0], [0, 0, 0, 1])
        pool.reset(b([0, 1, 0, 0]))
        with pytest.raises(RuntimeError, match="slot 2: its stream has ended"):
            pool.check()
        pool.reset(b([0, 0, 1, 0]))
        with pytest.raises(RuntimeError, match="slot 3: CQT pyramid"):
            pool.check()
        pool.reset()
        pool.check()


def test_launches_and_allocations_do_not_depend_on_the_mix():
    m = _v2()().cuda()
    S, chunk = 16, 4096
    pool = DevicePyramidPool(m, S, chunk)
    x = torch.randn(S, chunk, device="cuda")
    i32 = lambda v: torch.as_tensor(np.asarray(v), dtype=torch.int32).cuda()  # noqa: E731
    end = torch.zeros(S, dtype=torch.bool, device="cuda")
    mixes = [np.full(S, chunk), np.zeros(S), np.arange(S) * 200 + 17, np.r_[chunk, np.zeros(S - 1)]]
    ins = [i32(v) for v in mixes]
    with torch.no_grad():
        for _ in range(12):
            pool.push(x, ins[0])
        end_one = end.clone()
        end_one[3] = True
        ins_end = [(v, end) for v in ins] + [(ins[0], end_one)]
        torch.cuda.synchronize()
        launches, mem = [], []
        for v, e in ins_end:
            mem.append(torch.cuda.memory_allocated())
            before = _C.launch_count()
            pool.push(x, v, e)
            launches.append(_C.launch_count() - before)
        torch.cuda.synchronize()
        mem.append(torch.cuda.memory_allocated())
    assert len(set(launches)) == 1, launches
    assert len(set(mem)) == 1, mem


def test_simt_path_raises_at_construction(monkeypatch):
    m = _v2()().cuda()
    monkeypatch.setenv("NNAUDIO_B200_PATH", "simt")
    with pytest.raises(RuntimeError, match="no streamed tensor-core"):
        DevicePyramidPool(m, 4, 1000)


def test_cfg4_trace():
    """cfg4 (CQT2010v2, 88 bins, 22.05 kHz, hop 512): 64 slots, streams of 2-6 s in 10-40 ms packets, ~15 % idle
    slots, every ended stream bit for bit the whole-clip call; one replayed graph per tick."""
    m = _v2()().cuda()
    S, sr = 64, 22050
    chunk = sr * 4 // 100
    rng = np.random.default_rng(12)
    g = torch.Generator(device="cuda").manual_seed(12)
    L = rng.integers(sr * 2, sr * 6, size=S)
    xs = [torch.randn(int(n), device="cuda", generator=g) for n in L]
    with torch.no_grad():
        pool = DevicePyramidPool(m, S, chunk)
        graph, (x, lengths, end, restart) = _graph(pool, S, chunk, torch.float32)
        pos = np.zeros(S, np.int64)
        parts = [[] for _ in range(S)]
        checked = 0
        while (pos < L).any():
            n = int(rng.integers(sr // 100, chunk + 1))
            take = np.where(rng.random(S) < 0.15, 0, np.minimum(n, L - pos))
            fin = (pos + take == L) & (take > 0)
            x.fill_(float("nan"))
            for s in np.flatnonzero(take).tolist():
                x[s, :take[s]] = xs[s][pos[s]:pos[s] + take[s]]
            lengths.copy_(torch.as_tensor(take, dtype=torch.int32))
            end.copy_(torch.as_tensor(fin))
            graph.replay()
            counts = pool.counts.cpu().numpy()
            for s in np.flatnonzero(counts).tolist():
                parts[s].append(pool.frames[s:s + 1, :, :counts[s]].clone())
            pos += take
            for s in np.flatnonzero(fin).tolist():
                assert torch.equal(torch.cat(parts[s], 2), m(xs[s][None])), s
                checked += 1
        assert checked == S and pool.errors.count_nonzero().item() == 0


def test_mel_and_pyramid_front_ends_in_one_graph():
    """One captured tick feeds the same packets to a DeviceStreamPool Mel front end and a DevicePyramidPool; both
    equal their host pools tick by tick."""
    sr, S, chunk = 22050, 6, 3000
    mel = features.MelSpectrogram(sr=sr, n_fft=1024, hop_length=256, n_mels=80, verbose=False).cuda()
    cqt = _v2()().cuda()
    tr = _trace(S, chunk, 60, 3, min_end=30000)
    xs = _inputs(tr, S, chunk, torch.float32, 3)
    with torch.no_grad():
        a, b = DeviceStreamPool(mel, S, chunk), DevicePyramidPool(cqt, S, chunk)
        ha, hb = StreamPool(mel, S, _strict=True), PyramidPool(cqt, S)
        x = torch.zeros(S, chunk, device="cuda")
        lengths = torch.zeros(S, dtype=torch.int32, device="cuda")
        end = torch.zeros(S, dtype=torch.bool, device="cuda")
        restart = torch.zeros(S, dtype=torch.bool, device="cuda")

        def tick():
            a.reset(restart)
            b.reset(restart)
            a.push(x, lengths, end)
            b.push(x, lengths, end)

        tick()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            tick()
        ends = 0
        for i, (ln, en, rs) in enumerate(tr):
            if rs.any():
                ha.reset(np.flatnonzero(rs))
                hb.reset(np.flatnonzero(rs))
            oa, ob = ha.push(xs[i], ln, en), hb.push(xs[i], ln, en)
            x.copy_(xs[i])
            lengths.copy_(torch.as_tensor(ln, dtype=torch.int32))
            end.copy_(torch.as_tensor(en))
            restart.copy_(torch.as_tensor(rs))
            g.replay()
            for pool, out in ((a, oa), (b, ob)):
                counts = pool.counts.cpu().numpy()
                want = np.zeros(S, int)
                want[out.slots.numpy()] = out.counts.numpy()
                assert (counts == want).all(), (i, counts, want)
                for r, s in enumerate(out.slots.tolist()):
                    assert torch.equal(pool.frames[s, ..., :counts[s]], out.frames[r, ..., :counts[s]]), (i, s)
            ends += int(en.sum())
        assert ends >= 3 and a.errors.count_nonzero().item() == 0 and b.errors.count_nonzero().item() == 0
