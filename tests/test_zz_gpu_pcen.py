"""GPU: PCEN (nnaudio_b200.pcen) against its float64 reference (tests/pcen_domain.py).

* forward parity over batch, channel and frame counts (tile edges, one long single-stream case), scalar and
  per-channel parameters, inputs with zeros over 1e-10 .. 1e6;
* the expm1 / log1p form: elementwise relative error where u / bias <= 1e-3, with the float32 difference form
  shown failing the same bound;
* gradients of E and the four parameters against float64 autograd, alone and behind a trainable MelSpectrogram;
* run-twice determinism of outputs and gradients;
* route proof with torch.profiler: one PCEN kernel per inference call, only PCEN kernels in a training step;
* streaming bit for bit: random chunkings through PCENStream, a Mel StreamPool, and a DeviceStreamPool tick
  captured with PCENStream in one CUDA graph, each against the offline call.
"""
import re

import numpy as np
import pytest
import torch

import pcen_domain as pd
from nnaudio_b200 import features
from nnaudio_b200.pcen import PCEN, PCENStream
from nnaudio_b200.streaming import DeviceStreamPool, StreamPool

pytestmark = pytest.mark.gpu

EPS = 1e-6


def _module(kind, C, trainable=False):
    s, gain, bias, power = pd.parameters(kind, C)
    return PCEN(n_channels=C if kind == "channel" else None, s=s, gain=gain, bias=bias, power=power, eps=EPS,
                trainable=trainable).cuda()


def _ref(E, m):
    """float64 reference P (and u) of module ``m`` on the float32 numpy E."""
    prm = [getattr(m, n).detach().cpu().double().numpy() for n in pd.PARAMS]
    P, _, u = pd.reference(E, *prm, m.eps)
    return P, u


def _maxrel(got, ref):
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))


def _shapes():
    out = []
    for B in (1, 3, 256):
        for C in (1, 40, 80, 128, 257):
            Ts = (1, 65, 431) if B * C > 4096 else (1, 2, 63, 64, 65, 130, 431)
            out += [(B, C, T) for T in Ts]
    return out


@pytest.mark.parametrize("kind", ["scalar", "channel"])
@pytest.mark.parametrize("B,C,T", _shapes())
def test_forward_matches_float64(B, C, T, kind):
    E = pd.spectrogram(B, C, T, seed=B * 1000 + C * 7 + T)
    m = _module(kind, C)
    with torch.no_grad():
        P = m(torch.from_numpy(E).cuda()).cpu().numpy()
    ref, _ = _ref(E, m)
    assert P.shape == (B, C, T)
    assert _maxrel(P, ref) <= 1e-5, (B, C, T, kind, _maxrel(P, ref))


@pytest.mark.parametrize("kind", ["scalar", "channel"])
def test_forward_long_single_stream(kind):
    B, C, T = 1, 40, 120_000
    E = pd.spectrogram(B, C, T, seed=5)
    m = _module(kind, C)
    with torch.no_grad():
        P = m(torch.from_numpy(E).cuda()).cpu().numpy()
    ref, _ = _ref(E, m)
    assert _maxrel(P, ref) <= 1e-5


def test_empty_and_noncontiguous_inputs():
    m = _module("scalar", 4)
    with torch.no_grad():
        assert m(torch.zeros(2, 4, 0, device="cuda")).shape == (2, 4, 0)
        assert m(torch.zeros(0, 4, 9, device="cuda")).shape == (0, 4, 9)
        E = torch.from_numpy(pd.spectrogram(2, 9, 4, seed=3)).cuda()  # (B, T, C) viewed as (B, C, T)
        got = m(E.transpose(1, 2))
    ref, _ = _ref(E.transpose(1, 2).contiguous().cpu().numpy(), m)
    assert _maxrel(got.cpu().numpy(), ref) <= 1e-5
    with pytest.raises(ValueError):
        _module("channel", 40)(torch.zeros(1, 41, 5, device="cuda"))
    with pytest.raises(RuntimeError, match="float32"):
        m(torch.zeros(1, 4, 5, device="cuda", dtype=torch.float16))


@pytest.mark.parametrize("kind", ["scalar", "channel"])
def test_no_cancellation_where_u_is_small(kind):
    """Entries with u / bias <= 1e-3 (quiet channels) hold 1e-5 elementwise; the float32 difference form does not."""
    B, C, T = 4, 40, 300
    E = pd.spectrogram(B, C, T, seed=11, lo=-10, hi=-1, zeros=0.0)
    m = _module(kind, C)
    with torch.no_grad():
        P = m(torch.from_numpy(E).cuda()).cpu().numpy()
    ref, u = _ref(E, m)
    bias = pd._per_channel(m.bias.cpu(), C)[None, :, None]
    small = (u / bias <= 1e-3) & (ref > 0)
    assert small.sum() > 1000
    rel = np.abs(P - ref)[small] / ref[small]
    assert rel.max() <= 1e-5, rel.max()
    M32 = torch.from_numpy(pd.smoother(E, pd._per_channel(m.s.cpu(), C))).float().cuda()
    naive = pd.naive_fp32(torch.from_numpy(E).cuda(), M32, m.gain.cpu(), m.bias.cpu(), m.power.cpu(),
                          EPS).cpu().double().numpy()
    naive_rel = np.abs(naive - ref)[small] / ref[small]
    assert naive_rel.max() > 1e-5, "the test must bite: the difference form cancels here"


def _grads_vs_float64(B, C, T, kind, seed, lo=-6.0, hi=3.0):
    E = pd.spectrogram(B, C, T, seed=seed, lo=lo, hi=hi)
    m = _module(kind, C, trainable=True)
    W = torch.randn(B, C, T, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    Eg = torch.from_numpy(E).cuda().requires_grad_(True)
    P = m(Eg)
    P.backward(W.float().cuda())
    got = {"E": Eg.grad.double().cpu()}
    got.update({n: getattr(m, n).grad.double().cpu() for n in pd.PARAMS})
    Ed = torch.from_numpy(E).double().requires_grad_(True)
    prm = {n: getattr(m, n).detach().double().cpu().requires_grad_(True) for n in pd.PARAMS}
    (pd.reference_torch(Ed, *(prm[n] for n in pd.PARAMS), EPS) * W).sum().backward()
    want = {"E": Ed.grad}
    want.update({n: prm[n].grad for n in pd.PARAMS})
    return got, want


@pytest.mark.parametrize("kind", ["scalar", "channel"])
@pytest.mark.parametrize("B,C,T", [(1, 1, 1), (3, 40, 130), (2, 257, 65), (1, 8, 700)])
def test_gradients_match_float64_autograd(B, C, T, kind):
    got, want = _grads_vs_float64(B, C, T, kind, seed=B + C + T)
    for n in want:
        assert got[n].shape == want[n].shape, n
        err = _maxrel(got[n].numpy().reshape(-1), want[n].numpy().reshape(-1))
        assert err <= 1e-4, (n, err)


def test_gradients_through_trainable_mel():
    """MelSpectrogram(trainable_mel=True) -> PCEN(trainable=True): the mel basis and the PCEN parameters against
    float64 autograd through the same chain (the Mel graph of tests/train_domain.py)."""
    import train_domain as td

    torch.manual_seed(0)
    mel = features.MelSpectrogram(sr=16000, n_fft=512, hop_length=160, n_mels=40, trainable_mel=True,
                                  verbose=False).cuda()
    m = PCEN(n_channels=40, sr=16000, hop_length=160, trainable=True).cuda()
    x = torch.randn(2, 8000, generator=torch.Generator().manual_seed(3))
    P = m(mel(x.cuda()))
    W = torch.randn(P.shape, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    P.backward(W.float().cuda())
    leaves = td._leaves(mel, ["mel_basis"], "cpu")
    y, _ = td._mel(leaves, "", mel, x.double(), "mel_basis")
    prm = {n: getattr(m, n).detach().double().cpu().requires_grad_(True) for n in pd.PARAMS}
    (pd.reference_torch(y, *(prm[n] for n in pd.PARAMS), m.eps) * W).sum().backward()
    pairs = [("mel_basis", mel.mel_basis.grad, leaves["mel_basis"].grad)]
    pairs += [(n, getattr(m, n).grad, prm[n].grad) for n in pd.PARAMS]
    for n, g, w in pairs:
        err = _maxrel(g.double().cpu().numpy().reshape(-1), w.numpy().reshape(-1))
        assert err <= 1e-4, (n, err)


@pytest.mark.parametrize("kind", ["scalar", "channel"])
def test_run_twice_bit_identical(kind):
    B, C, T = 256, 128, 200
    E = torch.from_numpy(pd.spectrogram(B, C, T, seed=9)).cuda()
    g = torch.randn(B, C, T, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    runs = []
    for _ in range(2):
        m = _module(kind, C, trainable=True)
        Eg = E.clone().requires_grad_(True)
        P = m(Eg)
        P.backward(g)
        runs.append([P.detach(), Eg.grad] + [getattr(m, n).grad for n in pd.PARAMS])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type.name == "CUDA" and "memcpy" not in e.name.lower()
            and "memset" not in e.name.lower()]


def test_route_proof_with_profiler():
    B, C, T = 8, 80, 300
    E = torch.from_numpy(pd.spectrogram(B, C, T, seed=2)).cuda()
    m = _module("channel", C, trainable=True)
    with torch.no_grad():
        m(E)  # warm-up: module load
    with torch.no_grad():
        names = _kernels(lambda: m(E))
    assert len(names) == 1 and "pcen_forward_kernel" in names[0], names
    g = torch.randn(B, C, T, device="cuda")
    Eg = E.clone().requires_grad_(True)

    def step():
        m(Eg).backward(g)

    step()
    for p in m.parameters():
        p.grad = None
    Eg.grad = None
    names = _kernels(step)
    found = sorted(re.search(r"pcen_\w+?_kernel", n).group(0) if "pcen_" in n else n for n in names)
    assert found == ["pcen_backward_kernel", "pcen_forward_kernel", "pcen_param_reduce_kernel"], names


@pytest.mark.parametrize("kind", ["scalar", "channel"])
def test_random_chunkings_equal_offline(kind):
    B, C, T = 3, 40, 777
    E = torch.from_numpy(pd.spectrogram(B, C, T, seed=21)).cuda()
    m = _module(kind, C)
    rng = np.random.default_rng(0)
    with torch.no_grad():
        whole = m(E)
        for trial in range(3):
            st = PCENStream(m, B, n_channels=C)
            cuts = np.sort(rng.integers(0, T + 1, size=12))
            cuts = np.concatenate([[0], cuts, [cuts[-1]], [T]])  # a repeated cut: a 0-frame step
            parts = [st.step(E[:, :, a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
            assert torch.equal(torch.cat(parts, 2), whole), trial


def _mel():
    return features.MelSpectrogram(sr=16000, n_fft=512, hop_length=160, n_mels=80, verbose=False).cuda()


def test_stream_pool_then_pcen_equals_offline():
    """Ragged packets, slots that join late, ends and restarts through a Mel StreamPool, each PoolOutput through
    PCENStream.step(frames, counts, slots): every completed stream equals pcen(mel(x)) bit for bit."""
    S, chunk, ticks = 5, 700, 50
    mel, m = _mel(), _module("channel", 80)
    pool, st = StreamPool(mel, S), PCENStream(m, S)
    rng = np.random.default_rng(7)
    gen = torch.Generator(device="cuda").manual_seed(7)
    streams, rows, done = [[] for _ in range(S)], [[] for _ in range(S)], []
    total = np.zeros(S, int)
    start = rng.integers(0, 10, size=S)  # joins
    ended = np.zeros(S, bool)
    with torch.no_grad():
        for i in range(ticks):
            restart = ended.copy()
            if restart.any():
                pool.reset(np.flatnonzero(restart))
                st.reset(torch.as_tensor(restart).cuda())
                for s in np.flatnonzero(restart):
                    streams[s], rows[s], total[s] = [], [], 0
            ended[:] = False
            x = torch.randn(S, chunk, device="cuda", generator=gen)
            lengths = rng.integers(0, chunk + 1, size=S) * (rng.random(S) < 0.8) * (i >= start)
            total += lengths
            end = (total > 2000) & (rng.random(S) < 0.1)
            ended |= end
            out = pool.push(x, lengths, end)
            P = st.step(out.frames, out.counts, out.slots)
            for s in range(S):
                streams[s].append(x[s, :lengths[s]])
            for r, s in enumerate(out.slots.tolist()):
                c = int(out.counts[r])
                assert torch.count_nonzero(P[r, :, c:]).item() == 0
                rows[s].append(P[r:r + 1, :, :c].clone())
            for s in np.flatnonzero(end):
                done.append((torch.cat(streams[s]), torch.cat(rows[s], 2)))
        assert len(done) >= 4
        for x, got in done:
            assert torch.equal(got, m(mel(x[None]))), (got.shape,)


def test_device_pool_and_pcen_in_one_cuda_graph():
    """DeviceStreamPool.push -> PCENStream.step captured with masked resets in one CUDA graph and replayed: each
    completed stream equals pcen(mel(x)) bit for bit, and frames past the counts are exact zeros."""
    S, chunk, ticks = 6, 640, 60
    mel, m = _mel(), _module("scalar", 80)
    pool = DeviceStreamPool(mel, S, chunk)
    st = PCENStream(m, S, n_channels=80)
    x = torch.zeros(S, chunk, device="cuda")
    lengths = torch.zeros(S, dtype=torch.int32, device="cuda")
    end = torch.zeros(S, dtype=torch.bool, device="cuda")
    restart = torch.zeros(S, dtype=torch.bool, device="cuda")
    with torch.no_grad():
        pool.reset(restart), st.reset(restart)
        pool.push(x, lengths, end)
        st.step(pool.frames, pool.counts)  # eager warm-up tick (every slot idle)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            pool.reset(restart)
            st.reset(restart)
            pool.push(x, lengths, end)
            P = st.step(pool.frames, pool.counts)
        rng = np.random.default_rng(3)
        gen = torch.Generator(device="cuda").manual_seed(3)
        total, ended = np.zeros(S, int), np.zeros(S, bool)
        streams, rows, done = [[] for _ in range(S)], [[] for _ in range(S)], []
        for i in range(ticks):
            rs = ended.copy()
            total[rs] = 0
            ended[:] = False
            ln = rng.integers(0, chunk + 1, size=S) * (rng.random(S) < 0.8)
            total += ln
            en = (total > 2000) & (rng.random(S) < 0.08)
            ended |= en
            xs = torch.randn(S, chunk, device="cuda", generator=gen)
            x.copy_(xs), lengths.copy_(torch.as_tensor(ln, dtype=torch.int32)), end.copy_(torch.as_tensor(en))
            restart.copy_(torch.as_tensor(rs))
            g.replay()
            counts = pool.counts.cpu().numpy()
            for s in range(S):
                if rs[s]:
                    streams[s], rows[s] = [], []
                assert torch.count_nonzero(P[s, :, counts[s]:]).item() == 0
                streams[s].append(xs[s, :ln[s]])
                rows[s].append(P[s:s + 1, :, :counts[s]].clone())
                if en[s]:
                    done.append((torch.cat(streams[s]), torch.cat(rows[s], 2)))
        assert pool.errors.count_nonzero().item() == 0
        assert len(done) >= 4
        for xs, got in done:
            assert torch.equal(got, m(mel(xs[None]))), (got.shape,)
