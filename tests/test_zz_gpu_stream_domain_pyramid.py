"""The streamed CQT pyramids and inverse STFT across the offline domain matrices (-m gpu).

Pyramids: every pyramid_domain row through ``StreamingPyramid`` (threshold and ragged chunkings), ``PyramidPool`` and
``DevicePyramidPool``.  The concatenated frames equal ``module(x)`` bit for bit; every push that returns frames moves
the stream counters by the plan once, one octave route per octave and one FIR route per stage it launched, and no
offline counter; the lock-step output meets pyramid_domain's float64 bars.  A row on the CUDA-core plan has no
streamed route (the push raises, the device pool refuses it at construction); a row whose octaves frame at
different rates is refused at construction.

Inverse STFT: every ola_domain inverse row with hop <= n_fft through ``StreamingInverse`` on ragged frame pushes:
1e-6 of the peak against the offline inverse (both overlap-add with fp32 atomics), the ola bars against float64, and
each push's executed flops those of the overlap-add GEMM over its frames, K chunks included."""
import gc
import warnings

import numpy as np
import pytest
import torch

import ola_domain as od
import pyramid_domain as pd
import stream_domain as sd
from helpers import build, run_oracle
from nnaudio_b200 import _C, iSTFT
from nnaudio_b200.streaming import DevicePyramidPool, PyramidPool, StreamingInverse, StreamingPyramid
from test_zz_gpu_device_pyramid_pool import _inputs, _trace
from test_zz_gpu_ola_domain import _check as ola_check
from test_zz_gpu_ola_domain import _device_dft_kernels
from test_zz_gpu_pyramid_domain import _check as pyramid_check
from test_zz_gpu_pyramid_pool import _run as pool_schedule
from test_zz_gpu_stream_domain import _moved, _snapshot

pytestmark = pytest.mark.gpu


def _pyr_chunkings(sp, L, seed):
    """The first push that returns a frame ends one sample past the first threshold; then a zero-length push, one
    sample, a push longer than the top bank, and ragged pushes (StreamingPyramid's readiness rule)."""
    big = max(sp.widths) + 3 * sp.hop
    t1 = next((t for t in range(1, L) if sp._ready(t) > 0), None)
    if t1 is None:  # a stream shorter than the latency: every frame comes with the flush
        out = {"threshold": [L // 2, 0, L - L // 2]}
    else:
        head = [t1 - 1, 1, 0, 1, big]
        out = {"threshold": head + [L - sum(head)] if L > sum(head) else [t1 - 1, L - t1 + 1]}
    rng = np.random.default_rng(seed)
    sizes = []
    while sum(sizes) < L:
        sizes.append(int(min(rng.integers(0, 2 * big), L - sum(sizes))))
    out["ragged"] = sizes
    return out


def _free():
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", sd.PYRAMID)
def test_pyramid_stream_domain(name, monkeypatch):
    cls, ctor, B, near = pd.ROWS[name][:4]
    opts = pd.row_options(name)
    fmt, norm = opts["formats"][0], opts["norms"][0]
    fkw = dict(output_format=fmt, normalization_type=norm)
    if opts["path"] == "simt":
        monkeypatch.setenv("NNAUDIO_B200_PATH", "simt")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mod = build(cls, ctor).cuda()
    if not sd.pyramid_streams(mod):
        with pytest.raises(ValueError, match="frame at different rates"):
            StreamingPyramid(mod, B)
        return
    F, widths, hop, e, gen = sd.pyramid_geometry(mod)
    L = pd.valid_length(mod, near)
    sp = StreamingPyramid(mod, B, **fkw)
    assert (sp.generation, sp.hop, sp.widths) == (gen, hop, widths)
    pm = _C.PAD_REFLECT if sp._reflect else _C.PAD_CONSTANT
    gen_t = torch.Generator(device="cuda").manual_seed(len(name))
    try:
        if opts["path"] == "simt":
            with pytest.raises(RuntimeError, match="no streamed tensor-core pyramid plan"):
                sp.push(torch.zeros(B, 4096, device="cuda"))
            with pytest.raises(RuntimeError, match="no streamed tensor-core pyramid plan"):
                DevicePyramidPool(mod, 2, 1000, **fkw)
            return
        for cname, sizes in _pyr_chunkings(sp, L, len(name)).items():
            x = torch.randn(B, L, device="cuda", generator=gen_t)
            with torch.no_grad(), warnings.catch_warnings():
                warnings.simplefilter("ignore")
                want = mod(x, **fkw)
            sp = StreamingPyramid(mod, B, **fkw)
            parts, p = [], 0
            for n in sizes + [None]:
                flush = n is None
                plan, _ = _C.cqt_pyramid_chunk_plan(sp.received, sp.n_carry, sp.frames, n or 0, flush, widths, hop,
                                                    pm, e)
                before, T0 = _snapshot(), sp.frames
                with torch.no_grad(), warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    parts.append(sp.flush() if flush else sp.push(x[:, p:p + n]))
                T = sp.frames - T0
                mine, off, other = _moved(before, _C.ROUTES_PYR)
                want_r = sd.pyramid_push(F, widths, hop, B, gen == 2, sd.fir_stages_launched([plan])) if T else {}
                assert mine == want_r and not any(off) and not other, (name, cname, n, T, mine, want_r, off)
                p += n or 0
            y = torch.cat(parts, 2)
            assert torch.equal(y, want), (name, cname, float((y - want).nan_to_num().abs().max()))
            if cname == "ragged":
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    c = run_oracle(cls, mod, x.cpu().numpy(), dict(output_format="Complex", normalization_type=norm),
                                   dtype=np.float64)
                pyramid_check(y, c[..., 0] + 1j * c[..., 1], fmt, F, "stream_domain", f"{name} stream")
        _pyramid_pools(mod, name, fkw, F, widths, hop, e, gen, pm, L)
    finally:
        _free()


def _pyramid_pools(mod, name, fkw, F, widths, hop, e, gen, pm, L):
    S = 3
    pool = PyramidPool(mod, S, **fkw)
    advance = pool._advance

    def counted(chunk, lanes, A, T_max, count):
        before = _snapshot()
        out = advance(chunk, lanes, A, T_max, count)
        mine, off, other = _moved(before, _C.ROUTES_PYR)
        want = {}
        if A > 0 and T_max > 0:
            want = sd.pyramid_push(F, widths, hop, A, gen == 2, sd.fir_stages_launched(
                [sig for sig, _ in _C.cqt_pyramid_pool_plan(lanes, A, widths, hop, pm, e)]))
        assert mine == want and not any(off) and not other, (name, A, T_max, mine, want)
        return out
    pool._advance = counted
    gen_t = torch.Generator(device="cuda").manual_seed(len(name) + 1)
    streams = [[torch.randn(int(L * f), device="cuda", generator=gen_t) for f in (1.0, 0.6)] for _ in range(S)]
    done = pool_schedule(pool, streams, seed=len(name), max_n=max(widths) + 4 * hop)
    for per_slot in done:
        for x, y, _ in per_slot:
            with torch.no_grad(), warnings.catch_warnings():
                warnings.simplefilter("ignore")
                want = mod(x[None], **fkw)
            assert torch.equal(y, want), (name, "pyramid pool")
    chunk = 3000
    dp = DevicePyramidPool(mod, S, chunk, **fkw)
    n_stages = len(widths) - 1 + (e > 1)
    want_push = sd.pyramid_push(F, widths, hop, S, gen == 2, n_stages)
    ticks = 40
    tr = _trace(S, chunk, ticks, len(name), min_end=max(widths))
    xs = _inputs(tr, S, chunk, torch.float32, len(name))
    streams, rows, finished = [[] for _ in range(S)], [[] for _ in range(S)], []
    for i, (ln, en, rs) in enumerate(tr):
        dp.reset(torch.as_tensor(rs).cuda())
        before = _snapshot()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            dp.push(xs[i], torch.as_tensor(ln, dtype=torch.int32).cuda(), torch.as_tensor(en).cuda())
        mine, off, other = _moved(before, _C.ROUTES_PYR)
        assert mine == want_push and not any(off) and not other, (name, i, mine, want_push)
        counts = dp.counts.cpu().numpy()
        for s in range(S):
            assert not dp.frames[s, :, counts[s]:].any(), "frames past the counts are exact zeros"
            if rs[s]:
                streams[s], rows[s] = [], []
            streams[s].append(xs[i, s, :ln[s]])
            rows[s].append(dp.frames[s:s + 1, :, :counts[s]].clone())
            if en[s]:
                finished.append((torch.cat(streams[s]), torch.cat(rows[s], 2)))
    for x, y in finished:
        with torch.no_grad(), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = mod(x[None], **fkw)
        assert torch.equal(y, want), (name, "device pyramid pool")


@pytest.mark.parametrize("name", [n for n in sd.INVERSE if od.ISTFT_ROWS[n]["hop"] <= od.ISTFT_ROWS[n]["n_fft"]])
def test_inverse_stream_domain(name):
    row = od.ISTFT_ROWS[name]
    n_fft, hop, B, T, onesided, center = (row[k] for k in ("n_fft", "hop", "B", "T", "onesided", "center"))
    f_in = n_fft // 2 + 1 if onesided else n_fft
    length = od.length_of(row, T)
    X = np.random.RandomState(len(name) + 300).standard_normal((B, f_in, T, 2)).astype(np.float32)
    Xd = torch.from_numpy(X).cuda()
    try:
        if n_fft <= 2048:
            mod = iSTFT(n_fft=n_fft, hop_length=hop, window=row["window"], center=center, verbose=False).cuda()
            win = mod.window_mask.reshape(-1).float().cpu().numpy()
            with torch.no_grad():
                want = mod(Xd, onesided=onesided, length=length)
            make = lambda: StreamingInverse(mod, B, onesided=onesided)  # noqa: E731
        else:  # the module's float64 design is too large: the kernels are built on the device
            from scipy.signal import get_window
            win = get_window(row["window"], n_fft, fftbins=True).astype(np.float32)
            kc, ks = _device_dft_kernels(n_fft)
            packed = _C.pack_istft_basis(kc, ks, f_in, onesided)
            del kc, ks
            wind = torch.from_numpy(win).cuda()
            want = _C.istft_forward(Xd, packed, wind, n_fft, hop, center, length)
            make = lambda: sd.direct_inverse(packed, wind, n_fft, hop, center, onesided, B, "cuda")  # noqa: E731
        if length is not None and length < n_fft + hop * (T - 1) - (2 * (n_fft // 2) if center else 0):
            # a stream returns samples before it knows the length: flush() refuses one shorter than they are
            si = make()
            si.push(Xd)
            with pytest.raises(ValueError, match="shorter than the"):
                si.flush(length)
            length = None
            want = _C.istft_forward(Xd, packed, wind, n_fft, hop, center, None) if n_fft > 2048 else \
                mod(Xd, onesided=onesided, length=None)
        wss = od.istft_wss(win, hop, T, center, length)
        good = wss >= 1e-6 * wss.max()
        rng = np.random.default_rng(len(name))
        cuts = [1, 0] + [int(v) for v in rng.integers(0, 4, size=3 * T)] + [T]
        for sizes in ([T], cuts):
            si = make()
            parts, p = [], 0
            _C.profile_read_exec_flops()
            _C.profile_enable(True)
            try:
                for n in sizes:
                    n = min(n, T - p)
                    parts.append(si.push(Xd[:, :, p:p + n]))
                    flops = _C.profile_read_exec_flops()
                    assert flops == (sd.istft_push(B, n, n_fft, f_in) if n else 0), (name, n, flops)
                    p += n
                    if p == T:
                        break
                parts.append(si.flush(length))
                assert _C.profile_read_exec_flops() == 0
            finally:
                _C.profile_enable(False)
                _C.profile_read()
            y = torch.cat(parts, 1)
            assert y.shape == want.shape, (name, y.shape, want.shape)
            # 1e-6 of the peak where the window sum-square is not tiny, and on y * wss everywhere (the division
            # by a tiny wss magnifies the atomics' rounding, as the float64 bars below allow)
            dy, w_ = (y - want).cpu().numpy(), want.cpu().numpy()
            d = float(np.abs(dy[:, good]).max() / np.abs(w_[:, good]).max())
            dw = float(np.abs(dy * wss).max() / np.abs(w_ * wss).max())
            assert d <= 1e-6 and dw <= 1e-6, (name, sizes, d, dw)
        ref, _ = od.ref_istft(X, win, hop, center, onesided, length)
        yn = y.cpu().numpy().astype(np.float64)
        ola_check(yn[:, good], ref[:, good], "stream_domain_istft", name)
        ola_check(yn * wss, ref * wss, "stream_domain_istft", name + " y*wss")
    finally:
        _free()
