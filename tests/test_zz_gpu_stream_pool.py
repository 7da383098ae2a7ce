"""GPU: StreamPool against the offline module, a one-stream StreamingTransform, and the fp64 oracle.

Seeded ragged schedules with churn (slots idle, ending and restarting at different pushes): on the tensor-core
routes every completed stream's rows are bitwise ``module(x_s[None])`` and bitwise the frames a one-stream
``StreamingTransform`` gives for the same packet boundaries (``_strict=True``: the fused pool route ran).  The
CQT1992v2 tall kernel picks its balanced tile schedule from a launch's tile count, so its bitwise cases run on
the static schedule (``NNAB_TALL_BALANCE=0``) and its default schedule is held to 2e-6 of the peak.
"""
import numpy as np
import pytest
import torch

from helpers import rel_errors, run_oracle
from nnaudio_b200 import _C, features
from nnaudio_b200.streaming import StreamingTransform, StreamPool

pytestmark = pytest.mark.gpu

CASES = {
    "stft_r4_mag": (lambda: features.STFT(n_fft=1024, hop_length=256, verbose=False), {}, 16000),
    "stft_r4_complex": (lambda: features.STFT(n_fft=1024, hop_length=256, output_format="Complex",
                                              verbose=False), {}, 16000),
    "stft_r4_phase": (lambda: features.STFT(n_fft=1024, hop_length=256, output_format="Phase", verbose=False),
                      {}, 16000),
    "stft_r2_constant": (lambda: features.STFT(n_fft=512, hop_length=256, pad_mode="constant", verbose=False),
                         {}, 16000),
    "stft_uncentred": (lambda: features.STFT(n_fft=1024, hop_length=256, center=False, verbose=False), {}, 16000),
    "stft_hamming": (lambda: features.STFT(n_fft=512, hop_length=128, window="hamming", verbose=False), {}, 16000),
    "stft_hop100": (lambda: features.STFT(n_fft=512, hop_length=100, verbose=False), {}, 16000),
    "mel_fused": (lambda: features.MelSpectrogram(sr=16000, n_fft=512, hop_length=128, n_mels=80, verbose=False),
                  {}, 16000),
    "gammatone": (lambda: features.Gammatonegram(sr=16000, n_fft=512, hop_length=128, n_bins=64, verbose=False),
                  {}, 16000),
    "mfcc": (lambda: features.MFCC(sr=16000, n_mfcc=20, n_fft=512, hop_length=128, top_db=None, verbose=False),
             {}, 16000),
    "cqt1992v2": (lambda: features.CQT1992v2(sr=16000, hop_length=128, fmin=55, n_bins=60, verbose=False), {},
                  16000),
    "cqt1992v2_complex": (lambda: features.CQT1992v2(sr=16000, hop_length=128, fmin=55, n_bins=60,
                                                     output_format="Complex", verbose=False),
                          {"normalization_type": "wrap"}, 16000),
    "cqt1992": (lambda: features.CQT1992(sr=8000, hop_length=64, fmin=200, n_bins=24), {}, 8000),
}
ORACLE = ("stft_r4_mag", "mel_fused", "mfcc", "cqt1992v2", "cqt1992")


def run_schedule(pool, sr, seed, pushes=None, n_streams=2, max_packet=600, dtype=torch.float32, check=True):
    """Drive ``pool`` with a seeded ragged schedule: every slot runs ``n_streams`` streams of 0.5-1 s one after
    the other (a new one the push after the last ended), packets of 0..max_packet samples, some slots idle in
    every push.  Returns (x, packet sizes, frames) of every completed stream; with ``check``, every push's rows
    past their counts are verified to be exact zeros."""
    S, dev = pool.slots, pool.ring.device
    rng = np.random.default_rng(seed)
    gen = torch.Generator(device=dev).manual_seed(seed)
    lens = rng.integers(sr // 2, sr + 1, size=(S, n_streams))
    xs = [[torch.randn(int(L), device=dev, generator=gen).to(dtype) for L in row] for row in lens]
    k = np.zeros(S, int)          # stream index per slot
    pos = np.zeros(S, int)
    sizes = [[] for _ in range(S)]
    rows = [[] for _ in range(S)]
    restart = np.zeros(S, bool)
    done = []
    while (k < n_streams).any():
        if restart.any():
            pool.reset(np.flatnonzero(restart))
            restart[:] = False
        active = k < n_streams
        left = np.array([len(xs[s][k[s]]) - pos[s] if active[s] else 0 for s in range(S)])
        want = rng.integers(0, max_packet + 1, size=S) * (rng.random(S) < 0.7)
        lengths = np.minimum(want, left)
        end = active & (lengths == left) & (rng.random(S) < 0.8)
        n = int(lengths.max())
        chunk = torch.zeros(S, n, device=dev, dtype=dtype)
        for s in np.flatnonzero(lengths):
            chunk[s, :lengths[s]] = xs[s][k[s]][pos[s]:pos[s] + lengths[s]]
        out = pool.push(chunk, lengths, end)
        for i, (s, c) in enumerate(zip(out.slots.tolist(), out.counts.tolist())):
            if check:
                assert torch.count_nonzero(out.frames[i, :, c:]).item() == 0, "padded frames are exact zeros"
            rows[s].append(out.frames[i:i + 1, :, :c])
        for s in np.flatnonzero(active):
            sizes[s].append(int(lengths[s]))
        pos += lengths
        for s in np.flatnonzero(end):
            done.append((xs[s][k[s]], sizes[s], torch.cat(rows[s], 2)))
            sizes[s], rows[s] = [], []
            k[s] += 1
            pos[s] = 0
            restart[s] = True
    return done


def _one_stream(m, x, sizes, kw):
    st = StreamingTransform(m, 1, _strict=True, **kw)
    parts, p = [], 0
    for n in sizes:
        parts.append(st.push(x[None, p:p + n]))
        p += n
    parts.append(st.flush())
    return torch.cat(parts, 2)


@pytest.mark.parametrize("name", sorted(CASES))
def test_ragged_pool_equals_offline_and_one_stream_bitwise(name, monkeypatch):
    make, kw, sr = CASES[name]
    if name.startswith("cqt1992v2"):
        monkeypatch.setenv("NNAB_TALL_BALANCE", "0")
    torch.manual_seed(0)
    m = make().cuda()
    with torch.no_grad():
        done = run_schedule(StreamPool(m, 6, _strict=True, **kw), sr, seed=len(name) * 13)
        assert len(done) == 12
        for j, (x, sizes, got) in enumerate(done):
            ref = m(x[None], **kw)
            assert got.shape == ref.shape, (name, j)
            assert torch.equal(got, ref), (name, j, (got - ref).abs().max().item())
            if j < 3:
                assert torch.equal(got, _one_stream(m, x, sizes, kw)), (name, j)
    if name in ORACLE:
        x, _, got = done[0]
        want = run_oracle(type(m).__name__, m, x[None].cpu().numpy(), kw)
        emax, _ = rel_errors(got.cpu().numpy(), want)
        assert emax <= 1e-4, (name, emax)


def test_cqt1992v2_default_schedule_within_2e6():
    make, kw, sr = CASES["cqt1992v2"]
    m = make().cuda()
    with torch.no_grad():
        for x, _, got in run_schedule(StreamPool(m, 6, _strict=True), sr, seed=3, n_streams=1):
            ref = m(x[None])
            assert (got - ref).abs().max().item() <= 2e-6 * ref.abs().max().item()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("name", ["stft_r4_mag", "mel_fused", "cqt1992v2"])
def test_16bit_chunks_equal_upcast_offline(name, dtype, monkeypatch):
    make, kw, sr = CASES[name]
    monkeypatch.setenv("NNAB_TALL_BALANCE", "0")
    m = make().cuda()
    with torch.no_grad():
        for x, _, got in run_schedule(StreamPool(m, 6, _strict=True, **kw), sr, seed=11, n_streams=1, dtype=dtype):
            assert torch.equal(got, m(x[None].float(), **kw))


def test_concat_route_under_simt(monkeypatch):
    monkeypatch.setenv("NNAUDIO_B200_PATH", "simt")
    make, kw, sr = CASES["mel_fused"]
    m = make().cuda()
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="no fused pool route"):
            run_schedule(StreamPool(m, 4, _strict=True), sr, seed=1, n_streams=1)
        done = run_schedule(StreamPool(m, 4), sr, seed=1, n_streams=2)
        for x, _, got in done:
            ref = m(x[None])
            assert got.shape == ref.shape
            assert (got - ref).abs().max().item() <= 1e-6 * ref.abs().max().item()


def test_steady_pushes_do_not_synchronise():
    m = features.MelSpectrogram(sr=16000, n_fft=512, hop_length=128, n_mels=80, verbose=False).cuda()
    pool = StreamPool(m, 256, _strict=True)
    x = torch.randn(256, 480, device="cuda")
    rng = np.random.default_rng(0)
    with torch.no_grad():
        pool.push(x, np.full(256, 480))  # first push: any lazy init happens outside the checked window
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for i in range(20):
                lengths = rng.integers(160, 481, size=256) * (rng.random(256) < 0.8)
                end = np.zeros(256, bool)
                end[i] = True
                pool.push(x, lengths, end)
                pool.reset([i])
        finally:
            torch.cuda.set_sync_debug_mode(0)


@pytest.mark.parametrize("name", ["stft_r4_mag", "mel_fused", "mfcc", "cqt1992v2"])
def test_launches_are_the_offline_plan_plus_carry_and_mask(name):
    make, kw, sr = CASES[name]
    m = make().cuda()
    pool = StreamPool(m, 8, _strict=True, **kw)
    x = torch.randn(8, 3000, device="cuda")
    with torch.no_grad():
        pool.push(x, np.full(8, 3000))
        lengths = np.array([0, 700, 1, 0, 2000, 300, 0, 5])
        name_c, args = pool._st._args()
        before = _C.launch_count()
        out = pool.push(x, lengths)
        pushed = _C.launch_count() - before
        A, T_max = out.frames.shape[0], out.frames.shape[2]
        assert A > 0
        v = torch.randn(A, (T_max - 1) * pool.hop + pool.K, device="cuda")
        before = _C.launch_count()
        getattr(_C, name_c)(v, **dict(args, center=False))
        offline = _C.launch_count() - before
    assert pushed == offline + 2, (pushed, offline)


def test_serving_trace_256_slots_bitwise():
    """256 slots of 16 kHz Mel (n_fft 512, hop 128, 80 mels), packets of 160-480 samples with some slots idle in
    each push, about 1 % of the slots ending and restarting per push, streams of up to 10 s."""
    m = features.MelSpectrogram(sr=16000, n_fft=512, hop_length=128, n_mels=80, verbose=False).cuda()
    S, L = 256, 160000
    pool = StreamPool(m, S, _strict=True)
    rng = np.random.default_rng(7)
    gen = torch.Generator(device="cuda").manual_seed(7)
    cur = torch.randn(S, L, device="cuda", generator=gen)
    stop = rng.integers(L // 10, L + 1, size=S)  # staggered first streams
    pos = np.zeros(S, int)
    rows = [[] for _ in range(S)]
    checked = 0
    with torch.no_grad():
        for step in range(700):
            lengths = rng.integers(160, 481, size=S) * (rng.random(S) < 0.85)
            lengths = np.minimum(lengths, stop - pos)
            end = (pos + lengths >= stop) | ((rng.random(S) < 0.01) & (pos + lengths > 4000))
            idx = torch.as_tensor(pos, device="cuda")[:, None] + torch.arange(480, device="cuda")[None]
            chunk = torch.gather(cur, 1, idx.clamp(max=L - 1))
            out = pool.push(chunk, lengths, end)
            for i, (s, c) in enumerate(zip(out.slots.tolist(), out.counts.tolist())):
                rows[s].append(out.frames[i:i + 1, :, :c])
            pos += lengths
            for s in np.flatnonzero(end):
                ref = m(cur[s:s + 1, :pos[s]])
                got = torch.cat(rows[s], 2)
                assert torch.equal(got, ref), (step, s)
                checked += 1
                rows[s] = []
                cur[s] = torch.randn(L, device="cuda", generator=gen)
                pos[s] = 0
                stop[s] = L
            if end.any():
                pool.reset(np.flatnonzero(end))
    assert checked >= 500, checked
