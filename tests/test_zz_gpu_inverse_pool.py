"""GPU: InversePool against the offline inverse, a one-stream StreamingInverse, and the fp64 oracle.

Seeded ragged schedules with churn (slots idle, ending with and without ``length``, restarting): every completed
stream's samples must equal ``module(X_s[None])`` / ``module.inverse(X_s[None])`` and a one-stream
``StreamingInverse`` on the same packet boundaries to 1e-6 of the peak (every route overlap-adds with fp32
atomics, so none is bit-repeatable), and the oracle to 1e-4.  Frames past each row's count are NaN, so a read of
one would show; output rows past their counts must be exact zeros.
"""
import numpy as np
import pytest
import torch

from helpers import rel_errors
from nnaudio_b200 import _C, features
from nnaudio_b200.streaming import InversePool, StreamingInverse, StreamPool
from oracle import nnaudio_oracle as oracle

pytestmark = pytest.mark.gpu

CASES = {
    "istft_512_onesided": (lambda: features.iSTFT(n_fft=512, hop_length=128, verbose=False), True),
    "istft_512_twosided": (lambda: features.iSTFT(n_fft=512, hop_length=128, verbose=False), False),
    "istft_1024_onesided": (lambda: features.iSTFT(n_fft=1024, hop_length=256, verbose=False), True),
    "istft_1024_twosided": (lambda: features.iSTFT(n_fft=1024, hop_length=256, verbose=False), False),
    "istft_uncentred": (lambda: features.iSTFT(n_fft=512, hop_length=128, center=False, verbose=False), True),
    "istft_hop100": (lambda: features.iSTFT(n_fft=512, hop_length=100, verbose=False), True),
    "istft_hamming": (lambda: features.iSTFT(n_fft=512, hop_length=128, window="hamming", verbose=False), True),
    "stft_inverse": (lambda: features.STFT(n_fft=1024, hop_length=256, iSTFT=True, verbose=False), True),
}
ORACLE = ("istft_512_twosided", "istft_hop100", "stft_inverse")


def _offline(m, X, onesided, length):
    if isinstance(m, features.STFT):
        return m.inverse(X, onesided=onesided, length=length)
    return m(X, onesided=onesided, length=length)


def _kernels(m):
    return (m.kernel_cos_inv, m.kernel_sin_inv) if isinstance(m, features.STFT) else (m.kernel_cos, m.kernel_sin)


def run_schedule(pool, seed, n_streams=2, max_packet=8):
    """Every slot runs ``n_streams`` streams of 30-90 frames one after the other (a new one the push after the
    last ended), packets of 0..max_packet frames in a random row order, some slots idle in every push, about
    half the ends with a length.  Returns (X, length, packet sizes, samples) of every completed stream."""
    S, dev, f_in = pool.slots, pool.state.device, pool.f_in
    rng = np.random.default_rng(seed)
    gen = torch.Generator(device=dev).manual_seed(seed)
    Ts = rng.integers(30, 91, size=(S, n_streams))
    xs = [[torch.randn(1, f_in, int(T), 2, device=dev, generator=gen) for T in row] for row in Ts]
    k, pos = np.zeros(S, int), np.zeros(S, int)
    sizes, got = [[] for _ in range(S)], [[] for _ in range(S)]
    restart = np.zeros(S, bool)
    done = []
    while (k < n_streams).any():
        if restart.any():
            pool.reset(np.flatnonzero(restart))
            restart[:] = False
        active = k < n_streams
        left = np.array([xs[s][k[s]].shape[2] - pos[s] if active[s] else 0 for s in range(S)])
        counts = np.minimum(rng.integers(0, max_packet + 1, size=S) * (rng.random(S) < 0.7), left)
        end = active & (counts == left) & (rng.random(S) < 0.8)
        length = np.full(S, -1)
        for s in np.flatnonzero(end & (rng.random(S) < 0.5)):
            T = xs[s][k[s]].shape[2]
            ola = pool.n_fft + pool.hop * (T - 1)
            # at least what a one-stream push of the last packet returns before its flush
            least = int(pool._emit_end(np.array([T]))[0]) - pool.offset
            length[s] = int(rng.integers(least, ola + 100))
        rows = rng.permutation(np.flatnonzero(counts))
        t = int(counts.max()) + int(rng.integers(0, 3))
        X = torch.full((len(rows), f_in, t, 2), float("nan"), device=dev)
        for r, s in enumerate(rows):
            X[r, :, :counts[s]] = xs[s][k[s]][0, :, pos[s]:pos[s] + counts[s]]
        out = pool.push(X, rows, counts[rows], end, length)
        for i, (s, c) in enumerate(zip(out.slots.tolist(), out.counts.tolist())):
            assert torch.count_nonzero(out.samples[i, c:]).item() == 0, "rows past their counts are exact zeros"
            got[s].append(out.samples[i, :c])
        for s in np.flatnonzero(active):
            sizes[s].append(int(counts[s]))
        pos += counts
        for s in np.flatnonzero(end):
            done.append((xs[s][k[s]], None if length[s] < 0 else int(length[s]), sizes[s], torch.cat(got[s])))
            sizes[s], got[s] = [], []
            k[s] += 1
            pos[s] = 0
            restart[s] = True
    return done


def _one_stream(m, onesided, X, sizes, length):
    st = StreamingInverse(m, 1, onesided=onesided)
    parts, p = [], 0
    for c in sizes:
        parts.append(st.push(X[:, :, p:p + c]))
        p += c
    parts.append(st.flush(length))
    return torch.cat(parts, 1)[0]


@pytest.mark.parametrize("name", sorted(CASES))
def test_ragged_pool_equals_offline_one_stream_and_oracle(name):
    make, onesided = CASES[name]
    torch.manual_seed(0)
    m = make().cuda()
    with torch.no_grad():
        pool = InversePool(m, 6, onesided=onesided)
        done = run_schedule(pool, seed=len(name) * 17)
        assert len(done) == 12
        assert any(ln is None for _, ln, _, _ in done) and any(ln is not None for _, ln, _, _ in done)
        for j, (X, length, sizes, got) in enumerate(done):
            ref = _offline(m, X, onesided, length)[0]
            peak = ref.abs().max().item()
            assert got.shape == ref.shape, (name, j, got.shape, ref.shape)
            assert (got - ref).abs().max().item() <= 1e-6 * peak, (name, j)
            if j < 4:
                one = _one_stream(m, onesided, X, sizes, length)
                assert (got - one).abs().max().item() <= 1e-6 * peak, (name, j)
    if name in ORACLE:
        kc, ks = _kernels(m)
        for X, length, _, got in done[:2]:
            want = oracle.istft(X.cpu().numpy(), kc.cpu().numpy(), ks.cpu().numpy(), m.window_mask.cpu().numpy(),
                                m.stride, center=m.center, onesided=onesided, length=length)
            emax, _ = rel_errors(got[None].cpu().numpy(), want)
            assert emax <= 1e-4, (name, emax)


def test_stream_pool_to_inverse_pool_reconstructs_every_client():
    """The reference's STFT -> inverse round trip bound, per client, with both halves served by pools: 32 slots
    of 16 kHz audio in 160-480-sample packets, some idle, each slot's length set to its sample count."""
    stft = features.STFT(n_fft=512, hop_length=128, output_format="Complex", iSTFT=True, verbose=False).cuda()
    S = 32
    fwd, inv = StreamPool(stft, S, _strict=True), InversePool(stft, S)
    rng = np.random.default_rng(5)
    gen = torch.Generator(device="cuda").manual_seed(5)
    L = rng.integers(4000, 16001, size=S)
    x = torch.randn(S, int(L.max()), device="cuda", generator=gen)
    pos = np.zeros(S, int)
    parts = [[] for _ in range(S)]
    with torch.no_grad():
        while (pos < L).any():
            lengths = np.minimum(rng.integers(160, 481, size=S) * (rng.random(S) < 0.85), L - pos)
            end = (pos < L) & (pos + lengths >= L)
            idx = torch.as_tensor(pos, device="cuda")[:, None] + torch.arange(480, device="cuda")[None]
            chunk = torch.gather(x, 1, idx.clamp(max=x.shape[1] - 1))
            a = fwd.push(chunk, lengths, end)
            y = inv.push(a.frames * 0.5, a.slots, a.counts, end, np.where(end, L, -1))
            for i, (s, c) in enumerate(zip(y.slots.tolist(), y.counts.tolist())):
                parts[s].append(y.samples[i, :c])
            pos += lengths
    for s in range(S):
        recon = 2 * torch.cat(parts[s])
        assert recon.shape[0] == L[s]
        assert np.allclose(x[s, :L[s]].cpu(), recon.cpu(), rtol=1e-5, atol=1e-3), s


def test_inverse_pool_push_does_not_synchronise():
    m = features.iSTFT(n_fft=512, hop_length=128, verbose=False).cuda()
    S = 64
    pool = InversePool(m, S, onesided=True)
    X = torch.randn(S, 257, 4, 2, device="cuda")
    rng = np.random.default_rng(0)
    with torch.no_grad():
        pool.push(X, np.arange(S), np.full(S, 4))  # first push: any lazy init happens outside the checked window
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for i in range(20):
                counts = rng.integers(0, 5, size=S)
                counts[i] = max(counts[i], 1)
                end = np.zeros(S, bool)
                end[i] = True
                pool.push(X, np.arange(S), counts, end)
                pool.reset([i])
        finally:
            torch.cuda.set_sync_debug_mode(0)


def test_push_launches_seed_prep_gemm_and_finalize_whatever_the_mix():
    """The launches of a push do not depend on how many slots it serves: 2 lanes or 60."""
    m = features.iSTFT(n_fft=512, hop_length=128, verbose=False).cuda()
    pool = InversePool(m, 64, onesided=True)
    X = torch.randn(64, 257, 6, 2, device="cuda")
    launches = []
    with torch.no_grad():
        pool.push(X, np.arange(64), np.full(64, 6))
        for rows in (np.array([3, 40]), np.arange(60)):
            before = _C.launch_count()
            pool.push(X[:len(rows)], rows, np.full(len(rows), 5))
            launches.append(_C.launch_count() - before)
    assert launches[0] == launches[1] and launches[0] <= 8, launches
