"""GPU: DeviceStreamPool / DeviceInversePool against StreamPool / InversePool on the same seeded serving traces,
eagerly and as one CUDA graph replayed tick by tick with its inputs updated in place.

Every tick, row s of the device pool (up to its count) must equal StreamPool's row for slot s bit for bit (the
CQT1992v2 cases run on the static tall schedule, ``NNAB_TALL_BALANCE=0``, as in the StreamPool tests), rows past
their counts must be exact zeros, the replayed graph must equal the eager pushes bit for bit, and completed streams
must equal ``module(x)``.  The analysis -> gain -> synthesis tick is held to 1e-6 of each slot's peak against
StreamPool -> gain -> InversePool (the overlap-add uses fp32 atomics).
"""
import numpy as np
import pytest
import torch

from nnaudio_b200 import _C, features
from nnaudio_b200.streaming import DeviceInversePool, DeviceStreamPool, InversePool, StreamPool

pytestmark = pytest.mark.gpu

CASES = {
    "stft_r4_mag": (lambda: features.STFT(n_fft=1024, hop_length=256, verbose=False), {}),
    "stft_complex": (lambda: features.STFT(n_fft=512, hop_length=128, output_format="Complex", verbose=False), {}),
    "stft_r2_constant": (lambda: features.STFT(n_fft=512, hop_length=256, pad_mode="constant", verbose=False), {}),
    "stft_uncentred": (lambda: features.STFT(n_fft=1024, hop_length=256, center=False, verbose=False), {}),
    "stft_hop100": (lambda: features.STFT(n_fft=512, hop_length=100, verbose=False), {}),
    "mel_fused": (lambda: features.MelSpectrogram(sr=16000, n_fft=512, hop_length=128, n_mels=80, verbose=False),
                  {}),
    "gammatone": (lambda: features.Gammatonegram(sr=16000, n_fft=512, hop_length=128, n_bins=64, verbose=False),
                  {}),
    "mfcc": (lambda: features.MFCC(sr=16000, n_mfcc=20, n_fft=512, hop_length=128, top_db=None, verbose=False), {}),
    "cqt1992v2": (lambda: features.CQT1992v2(sr=16000, hop_length=128, fmin=55, n_bins=60, verbose=False), {}),
    "cqt1992": (lambda: features.CQT1992(sr=8000, hop_length=64, fmin=200, n_bins=24), {}),
}


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
        end = (total > min_end) & (rng.random(S) < 0.08)
        ended |= end
        out.append((lengths, end, restart))
    return out


def _inputs(S, chunk, dtype, ticks, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(ticks, S, chunk, device="cuda", generator=gen).to(dtype)


def _run(make, kw, dtype, S=6, ticks=60, seed=0):
    m = make().cuda()
    host = StreamPool(m, S, _strict=True, **kw)
    chunk = max(400, host.K // 8)  # long CQT kernels: streams that reach an end within the trace
    tr = _trace(S, chunk, ticks, seed, min_end=host.K)
    xs = _inputs(S, chunk, dtype, ticks, seed)
    eager = DeviceStreamPool(m, S, chunk, dtype, **kw)
    graphed = DeviceStreamPool(m, S, chunk, dtype, **kw)
    x = torch.zeros(S, chunk, device="cuda", dtype=dtype)
    lengths = torch.zeros(S, dtype=torch.int32, device="cuda")
    end = torch.zeros(S, dtype=torch.bool, device="cuda")
    restart = torch.zeros(S, dtype=torch.bool, device="cuda")
    graphed.reset(restart)
    graphed.push(x, lengths, end)  # eager warm-up tick (every slot idle)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        graphed.reset(restart)
        graphed.push(x, lengths, end)
    streams = [[] for _ in range(S)]
    rows = [[] for _ in range(S)]
    done = []
    for i, (ln, en, rs) in enumerate(tr):
        dev_in = (torch.as_tensor(ln, dtype=torch.int32).cuda(), torch.as_tensor(en).cuda(),
                  torch.as_tensor(rs).cuda())
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
        x.copy_(xs[i]), lengths.copy_(dev_in[0]), end.copy_(dev_in[1]), restart.copy_(dev_in[2])
        g.replay()
        assert torch.equal(graphed.frames, eager.frames) and torch.equal(graphed.counts, eager.counts), i
        counts = eager.counts.cpu().numpy()
        want = np.zeros(S, int)
        want[out.slots.numpy()] = out.counts.numpy()
        assert (counts == want).all(), (i, counts, want)
        for r, s in enumerate(out.slots.tolist()):
            assert torch.equal(eager.frames[s, :, :counts[s]], out.frames[r, :, :counts[s]]), (i, s)
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
    return m, done


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("name", sorted(CASES))
def test_device_pool_equals_stream_pool_eager_and_graph(name, dtype, monkeypatch):
    if name == "cqt1992v2":
        monkeypatch.setenv("NNAB_TALL_BALANCE", "0")
    make, kw = CASES[name]
    with torch.no_grad():
        m, done = _run(make, kw, dtype, seed=len(name))
        assert len(done) >= 3
        for x, got in done[:3]:
            ref = m(x[None].float(), **kw)
            assert torch.equal(got, ref), (name, (got - ref).abs().max().item())


def test_errors_drop_the_slot_and_check_raises_the_host_type():
    m = features.MelSpectrogram(sr=16000, n_fft=512, hop_length=128, n_mels=80, verbose=False).cuda()
    S, chunk = 4, 300
    pool = DeviceStreamPool(m, S, chunk)
    x = torch.randn(S, chunk, device="cuda")
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")
    b = lambda v: torch.tensor(v, dtype=torch.bool, device="cuda")
    with torch.no_grad():
        pool.push(x, i32([300, 300, 300, 0]), b([0, 0, 1, 0]))
        before = pool.counters.clone()
        pool.push(x, i32([300, 301, 100, 0]), b([0, 0, 0, 1]))  # slot 1: too long, 2: ended, 3: too short
        assert pool.errors.tolist() == [0, _C.LANE_ELENGTH, _C.LANE_EENDED, _C.LANE_ESHORT]
        assert torch.equal(pool.counters[:, 1:], before[:, 1:]), "dropped slots keep their counters"
        assert pool.counters[0, 0].item() == 600
        assert pool.counts[1:].count_nonzero().item() == 0 and pool.frames[1:].count_nonzero().item() == 0
        with pytest.raises(ValueError, match="slot 1 has 301"):
            pool.check()
        host = StreamPool(m, S)
        with pytest.raises(ValueError, match="slot 1 has 301"):
            host.push(x, [300, 301, 100, 0], [0, 0, 0, 1])
        pool.reset(b([0, 1, 0, 0]))
        with pytest.raises(RuntimeError, match="slot 2: its stream has ended"):
            pool.check()
        pool.reset(b([0, 0, 1, 0]))
        with pytest.raises(AssertionError, match="slot 3: Signal length shorter"):
            pool.check()
        pool.reset()
        pool.check()
        inv = DeviceInversePool(features.STFT(n_fft=512, hop_length=128, iSTFT=True, verbose=False).cuda(), S, 4)
        X = torch.randn(S, 257, 4, 2, device="cuda")
        inv.push(X, i32([0, 5, 2, 0]), b([1, 0, 0, 0]))
        assert inv.errors.tolist() == [_C.LANE_ENOFRAMES, _C.LANE_ELENGTH, 0, 0]
        with pytest.raises(RuntimeError, match="slot 0: ending a stream without frames"):
            inv.check()


def test_construction_and_argument_refusals(monkeypatch):
    m = features.MelSpectrogram(sr=16000, n_fft=512, hop_length=128, n_mels=80, verbose=False).cuda()
    pool = DeviceStreamPool(m, 4, 300)
    x = torch.randn(4, 300, device="cuda")
    ok_len = torch.zeros(4, dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError):
        pool.push(x[:, :200], ok_len)
    with pytest.raises(ValueError):
        pool.push(x.half(), ok_len)
    with pytest.raises(RuntimeError):
        pool.push(x.cpu(), ok_len)
    with pytest.raises(TypeError):
        pool.push(x, ok_len.cpu())
    with pytest.raises(TypeError):
        pool.push(x, ok_len.long())
    with pytest.raises(ValueError):
        pool.push(x, ok_len[:3])
    with pytest.raises(TypeError):
        pool.push(x, [0, 0, 0, 0])
    monkeypatch.setenv("NNAUDIO_B200_PATH", "simt")
    with pytest.raises(RuntimeError, match="no fused pool route"):
        DeviceStreamPool(m, 4, 300)


def test_analysis_gain_synthesis_graph_matches_host_pools():
    stft = features.STFT(n_fft=512, hop_length=128, output_format="Complex", iSTFT=True, verbose=False).cuda()
    S, chunk, ticks, gain = 8, 480, 80, 0.5
    tr = _trace(S, chunk, ticks, 5, min_end=512)
    xs = _inputs(S, chunk, torch.float32, ticks, 5)
    with torch.no_grad():
        fwd, inv = StreamPool(stft, S, _strict=True), InversePool(stft, S)
        pool = DeviceStreamPool(stft, S, chunk)
        syn = DeviceInversePool(stft, S, frames=pool.T_cap)
        x = torch.zeros(S, chunk, device="cuda")
        lengths = torch.zeros(S, dtype=torch.int32, device="cuda")
        end = torch.zeros(S, dtype=torch.bool, device="cuda")
        restart = torch.zeros(S, dtype=torch.bool, device="cuda")
        length = torch.full((S,), -1, dtype=torch.int64, device="cuda")

        def tick():
            pool.reset(restart)
            syn.reset(restart)
            pool.push(x, lengths, end)
            syn.push(pool.frames * gain, pool.counts, end, length)

        tick()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            tick()
        got = [[] for _ in range(S)]
        want = [[] for _ in range(S)]
        checked = 0
        for i, (ln, en, rs) in enumerate(tr):
            if rs.any():
                fwd.reset(np.flatnonzero(rs))
                inv.reset(np.flatnonzero(rs))
            a = fwd.push(xs[i], ln, en)
            y = inv.push(a.frames * gain, a.slots, a.counts, en)
            x.copy_(xs[i])
            lengths.copy_(torch.as_tensor(ln, dtype=torch.int32))
            end.copy_(torch.as_tensor(en))
            restart.copy_(torch.as_tensor(rs))
            g.replay()
            counts = syn.counts.cpu().numpy()
            for r, (s, c) in enumerate(zip(y.slots.tolist(), y.counts.tolist())):
                want[s].append(y.samples[r, :c])
            for s in range(S):
                assert syn.samples[s, counts[s]:].count_nonzero().item() == 0
                got[s].append(syn.samples[s, :counts[s]].clone())
            for s in np.flatnonzero(en):
                a_, b_ = torch.cat(got[s]), torch.cat(want[s])
                assert a_.shape == b_.shape, (i, s)
                assert (a_ - b_).abs().max().item() <= 1e-6 * b_.abs().max().item(), (i, s)
                got[s], want[s] = [], []
                checked += 1
        assert checked >= 5 and syn.errors.count_nonzero().item() == 0
