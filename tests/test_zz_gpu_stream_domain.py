"""The streamed forward transforms across the offline domain matrices (-m gpu): every row of tests/stream_domain.py
(dense_domain, cqt1992_domain, block_domain's module shapes and three stream-only edges) through
``StreamingTransform``, ``StreamPool`` and ``DeviceStreamPool``.

- Lock-step pushes over every chunking the row's readiness thresholds give: the concatenated frames equal the
  offline call bit for bit; every push moves the stream route counters (``_C.stream_route_count``) and the
  executed-MMA-flop counter exactly as the offline model of its virtual clip predicts, and no offline counter.
- One seeded ragged ``StreamPool`` schedule with churn and one ``DeviceStreamPool`` trace per row: every completed
  stream bit for bit its offline call, frames past the counts exact zeros, counter deltas as modelled.
- On one chunking the stream meets the row's float64 bars: 1e-4 max-relative and L2-relative, 1e-3 per bin, filter
  or 8-bin group, 2e-3 in phase.
- Known exceptions: the CQT1992v2 tall kernel's bitwise runs use its static schedule (``NNAB_TALL_BALANCE=0``) and
  its default schedule is held to 2e-6 of the peak; rows whose plan is the CUDA-core kernel have no fused chunk
  route: ``_strict`` pushes raise, the concat route matches offline to 1e-6 of the peak and moves the offline SIMT
  counter, and the device pool refuses them at construction.
- bf16 and fp16 chunks equal the fp32 upcast bit for bit on one row per tensor-core route."""
import gc
import os
import warnings

import numpy as np
import pytest
import torch

import dense_domain as dd
import stream_domain as sd
from conftest import record_error
from helpers import build, run_oracle
from nnaudio_b200 import _C
from nnaudio_b200.streaming import DeviceStreamPool, StreamingTransform, StreamPool
from test_zz_gpu_dense_domain import _device_basis
from test_zz_gpu_device_pool import _inputs, _trace
from test_zz_gpu_stream_pool import run_schedule

pytestmark = pytest.mark.gpu

BAR, GROUP_BAR, PHASE_FLOOR, PHASE_BAR = 1e-4, 1e-3, 0.01, 2e-3
FMT_IDS = {"Complex": _C.FMT_COMPLEX, "Magnitude": _C.FMT_MAGNITUDE, "Phase": _C.FMT_PHASE_ANGLE}
# one row per tensor-core route for the 16-bit chunks
HALF_ROWS = ("block:512_128", "dense:hamming_rows", "dense:splitk_8192", "dense:mel_fused_speech",
             "dense:gammatone_planes", "dense:mel_3_sums", "cqt:tall_base", "cqt:varn_hop96_k4096",
             "cqt:varn_hop64", "cqt:dense_k2048", "cqt:dense_hop100")


def _snapshot():
    fams = ((_C.ROUTES_STFT, _C.STFT_ROUTES), (_C.ROUTES_CQ1992, _C.CQ1992_ROUTES), (_C.ROUTES_PYR, _C.PYR_ROUTES))
    stream = {(f, r): _C.stream_route_count(f, r) for f, n in fams for r in range(n)}
    offline = ([_C.stft_route_count(r) for r in range(_C.STFT_ROUTES)]
               + [_C.cqt1992v2_route_count(r) for r in range(_C.CQ1992_ROUTES)]
               + [_C.pyramid_route_count(r) for r in range(_C.PYR_ROUTES)])
    return stream, offline


def _moved(before, fam):
    """({route: delta} of family ``fam``'s stream counters, offline counter deltas, other stream deltas)."""
    s0, o0 = before
    s1, o1 = _snapshot()
    mine = {r: s1[(f, r)] - s0[(f, r)] for (f, r) in s1 if f == fam and s1[(f, r)] != s0[(f, r)]}
    other = {k: s1[k] - s0[k] for k in s1 if k[0] != fam and s1[k] != s0[k]}
    return mine, [b - a for a, b in zip(o0, o1)], other


class Row:
    """A forward row on the device: offline call, stream and pool factories, the push model, the float64 check."""

    def __init__(self, name):
        self.name = name
        self.cls = sd.base_class(name)
        self.opts = sd.options(name)
        self.stft = sd.is_stft(name)
        self.fam = _C.ROUTES_STFT if self.stft else _C.ROUTES_CQ1992
        self.fmt = self.opts["formats"][0]
        self.simt = sd.auto_simt(name)
        self.fb = None
        dev = "cuda"
        if sd.is_direct(name):
            ctor = sd.constructor(name)
            K, hop = ctor["n_fft"], ctor["hop_length"]
            self.win = dd.window(ctor.get("window", "hann"), K)
            wcos, wsin = _device_basis(K, self.win)
            kw = dict(wcos=wcos, wsin=wsin, packed=_C.pack_basis(wcos, wsin), n_fft=K, hop=hop,
                      center=ctor.get("center", True), pad_mode=_C.PAD_REFLECT)
            if self.cls == "STFT":
                self.call, kw = "stft_forward", dict(kw, out_format=FMT_IDS[self.fmt], sqrt_eps=0.0)
            else:
                self.fb = sd.bank(name)
                fb = torch.from_numpy(self.fb.astype(np.float32)).cuda()
                self.call = "stft_filterbank_forward"
                kw = dict(kw, sqrt_eps=0.0, power=2.0, fb=fb, fb_table=_C.build_filterbank_table(fb))
            self.kw = kw
            self.offline = lambda x: getattr(_C, self.call)(x, **kw)
            self.stream = lambda B: sd.direct_stream(name, kw, B, dev)
            self.mod = None
        else:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                self.mod = mod = build(self.cls, sd.constructor(name)).cuda()
            if self.opts.get("nudge"):
                with torch.no_grad():
                    g = torch.Generator(device="cpu").manual_seed(7)
                    mod.wcos.add_(self.opts["nudge"] * torch.randn(mod.wcos.shape, generator=g).cuda())
                    mod.wsin.add_(self.opts["nudge"] * torch.randn(mod.wsin.shape, generator=g).cuda())
            self.fkw = {}
            if self.cls in ("STFT", "CQT1992v2", "CQT"):
                self.fkw["output_format"] = self.fmt
            if not self.stft:
                self.fkw["normalization_type"] = self.opts["norms"][0]
            if self.cls in ("MelSpectrogram", "MFCC", "Gammatonegram"):
                mel = mod.melspec_layer if self.cls == "MFCC" else mod
                self.fb = (mel.gammatone_basis if self.cls == "Gammatonegram" else mel.mel_basis).detach().cpu().numpy()
            self.offline = lambda x: mod(x, **self.fkw)
            self.stream = lambda B: StreamingTransform(mod, B, _strict=not self.simt, **self.fkw)
        K = self.mod.kernel_width if self.mod is not None and not self.stft else None
        self.K, self.hop, self.pad, self.reflect = sd.geometry(name, K)
        self.chunkings = sd.row_chunkings(name, K)

    def model(self, A, T, balance=True, tall_ctas=None, passes=3):
        """(stream counter deltas, flops) of a push of A rows, T_max frames."""
        if self.stft:
            p = sd.stft_push(self.name, A, T, self.fb, passes)
            return p["routes"], p["flops"]
        p = sd.cq1992_push(self.mod, A, T, balance, tall_ctas)
        return {p["route"]: 1}, p["flops"]

    def host_pool(self, slots):
        if self.mod is not None:
            return StreamPool(self.mod, slots, _strict=not self.simt, **self.fkw)
        pool = StreamPool.__new__(StreamPool)  # the direct basis: StreamPool on a direct_stream (stream_domain)
        pool._st = st = self.stream(slots)
        pool.module, pool._strict = None, False
        pool.K, pool.hop, pool.pad, pool._reflect, pool.ring = st.K, st.hop, st.pad, st._reflect, st.ring
        pool._init_slots(slots)
        pool.dtype = None
        return pool

    def check_float64(self, y, xn):
        """The row's float64 bars on the stream's output y (numpy) for input xn; returns the worst errors."""
        if not self.stft:
            c = run_oracle(self.cls, self.mod, xn, dict(output_format="Complex",
                                                        normalization_type=self.opts["norms"][0]), dtype=np.float64)
            return _bars(y, c[..., 0] + 1j * c[..., 1], self.fmt, 8, self.name)
        center = self.pad > 0
        pm = "reflect" if self.reflect or not center else "constant"
        if self.mod is None:
            X = dd.ref_stft_fft(xn, self.win, self.hop, center, pm)
        else:
            stft = self.mod if self.cls == "STFT" else (self.mod.melspec_layer.stft if self.cls == "MFCC"
                                                        else self.mod.stft)
            X = dd.ref_stft(xn, stft.wcos.detach().cpu().numpy(), stft.wsin.detach().cpu().numpy(), self.hop,
                            center, pm)
        if self.cls == "STFT":
            return _bars(y, X, self.fmt, 1, self.name, trainable=bool(self.opts.get("nudge")))
        trainable = self.mod is not None and bool(sd.constructor(self.name).get("trainable", False))
        power = 2.0 if self.mod is None else float((self.mod.melspec_layer if self.cls == "MFCC" else self.mod).power)
        S = dd.ref_filterbank(X, self.fb.astype(np.float64), power, trainable)
        if self.cls == "MFCC":
            S = dd.ref_mfcc(S, self.mod.n_mfcc, self.mod._amin_host, self.mod._ref_host, None)
            return _bars(y, S, "Magnitude", None, self.name)
        return _bars(y, S, "Magnitude", 1, self.name)


def _bars(y, X, fmt, group, name, trainable=False):
    """Global bars, per bin / filter (group 1), per 8-bin group (8) or none (None), and phase."""
    y = np.asarray(y, dtype=np.float64)
    mag = np.abs(X)
    if fmt == "Phase":
        mask = mag > PHASE_FLOOR * mag.max()
        got = np.exp(1j * y) if y.ndim == 3 else y[..., 0] + 1j * y[..., 1]
        d = float(np.abs(got - X / np.where(mag > 0, mag, 1))[mask].max())
        record_error("stream_domain", name, phase_unit_max=d)
        assert d <= PHASE_BAR, (name, d)
        return dict(phase=d)
    if fmt == "Complex":
        got, want = y[..., 0] + 1j * y[..., 1], X
    else:
        got, want = y, (np.sqrt(mag ** 2 + 1e-8) if trainable else mag) if np.iscomplexobj(X) else X
    d = np.abs(got - want)
    scale = np.abs(want)
    emax = float(d.max() / scale.max())
    el2 = float(np.linalg.norm(d) / np.linalg.norm(scale))
    out = dict(max_rel=emax, l2_rel=el2)
    if group:
        n = d.shape[1]
        per = [float(d[:, i:i + group].max() / max(np.sqrt((scale[:, i:i + group] ** 2).mean()), 1e-30))
               for i in range(0, n, group)]
        out["group"] = max(per)
        assert out["group"] <= GROUP_BAR, (name, int(np.argmax(per)), out)
    record_error("stream_domain", name, **out)
    assert emax <= BAR and el2 <= BAR, (name, out)
    return out


def _cat(parts):
    return torch.cat(parts, 2)


def _lock_step(row, x, sizes, balance, tall_ctas, flops_passes=3):
    """Push ``sizes`` then flush through a fresh stream of row; every push's counters against the model."""
    st = row.stream(x.shape[0])
    parts, p = [], 0
    _C.profile_read_exec_flops()
    for n in list(sizes) + [None]:
        before = _snapshot()
        T0 = st.frames
        with torch.no_grad(), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            y = st.flush() if n is None else st.push(x[:, p:p + n])
        flops = _C.profile_read_exec_flops()
        T = st.frames - T0
        mine, off, other = _moved(before, row.fam)
        assert not other, (row.name, other)
        if row.simt:
            simt = _C.STFT_SIMT if row.stft else _C.STFT_ROUTES + _C.CQ1992_SIMT
            want_off = [0] * len(off)
            if T > 0:
                want_off[simt] = 1
                if row.fb is not None:
                    want_off[_C.STFT_FB_GEMM] = 1
            assert not mine and off == want_off, (row.name, n, mine, off)
        else:
            want, want_flops = row.model(x.shape[0], T, balance, tall_ctas, flops_passes) if T > 0 else ({}, 0.0)
            assert mine == want, (row.name, n, T, mine, want)
            assert flops == want_flops, (row.name, n, T, flops, want_flops)
            assert not any(off), (row.name, n, "an offline counter moved", off)
        parts.append(y)
        p += n or 0
    return _cat(parts)


def _free():
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", sd.FORWARD)
def test_stream_domain(name, monkeypatch):
    opts = sd.options(name)
    if opts["path"] == "simt":
        monkeypatch.setenv("NNAUDIO_B200_PATH", "simt")
    tall_ctas = next((c for c in opts.get("tall_ctas", (None,)) if c), None)
    if tall_ctas:
        monkeypatch.setenv("NNAB_TALL_CTAS", str(tall_ctas))
    _C.profile_enable(True)
    try:
        row = Row(name)
        B = sd.clip(name)[0]
        tall = not row.stft and sd.CQ_ROWS[name][5] in (_C.CQ1992_TALL, _C.CQ1992_TALL_BALANCED)
        monkeypatch.setenv("NNAB_TALL_BALANCE", "0")  # the tall kernel's static schedule: bitwise
        gen = torch.Generator(device="cuda").manual_seed(len(name))
        f64_chunking = "ragged" if "ragged" in row.chunkings else "threshold"
        for cname, sizes in row.chunkings.items():
            x = torch.randn(B, sum(sizes), device="cuda", generator=gen)
            with torch.no_grad(), warnings.catch_warnings():
                warnings.simplefilter("ignore")
                want = row.offline(x)
            y = _lock_step(row, x, sizes, False, tall_ctas)
            assert y.shape == want.shape, (name, cname, y.shape, want.shape)
            if row.simt:
                d = float((y - want).abs().max() / want.abs().max())
                assert d <= 1e-6, (name, cname, d)
            else:
                assert torch.equal(y, want), (name, cname, float((y - want).nan_to_num().abs().max()))
            if cname == f64_chunking:
                errs = row.check_float64(y.cpu().numpy(), x.cpu().numpy())
                print(f"{name} [{cname}] float64 " + " ".join(f"{k} {v:.2e}" for k, v in errs.items()))
        if row.simt:
            st = row.stream(B)
            st._strict = True
            with pytest.raises(RuntimeError, match="no fused chunk route"):
                st.push(torch.zeros(B, row.K + row.hop, device="cuda"))
        if tall:  # the default (balanced when it pays) schedule: routes as modelled, 2e-6 of the peak
            monkeypatch.delenv("NNAB_TALL_BALANCE")
            sizes = row.chunkings["threshold"]
            x = torch.randn(B, sum(sizes), device="cuda", generator=gen)
            with torch.no_grad():
                want = row.offline(x)
            y = _lock_step(row, x, sizes, True, tall_ctas)
            d = float((y - want).abs().max() / want.abs().max())
            assert d <= 2e-6, (name, d)
            monkeypatch.setenv("NNAB_TALL_BALANCE", "0")
        _pools(row, gen)
        if name in HALF_ROWS:
            _half(row, gen, B, tall_ctas)
    finally:
        _C.profile_enable(False)
        _C.profile_read()
        row = None
        _free()


def _check_pool_push(row, out, before):
    mine, off, other = _moved(before, row.fam)
    assert not other, (row.name, other)
    A = len(out.slots)
    if row.simt:
        simt = _C.STFT_SIMT if row.stft else _C.STFT_ROUTES + _C.CQ1992_SIMT
        assert not mine and off[simt] == (1 if A else 0), (row.name, mine, off)
        return
    T_max = out.frames.shape[2]
    want = row.model(A, T_max, False)[0] if A else {}
    assert mine == want and not any(off), (row.name, A, T_max, mine, want, off)


def _pools(row, gen):
    """One ragged StreamPool schedule with churn and one DeviceStreamPool trace."""
    S = 3
    pool = row.host_pool(S)
    push = pool.push

    def counted(chunk, lengths, end=None):
        before = _snapshot()
        with torch.no_grad(), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out = push(chunk, lengths, end)
        _check_pool_push(row, out, before)
        return out
    pool.push = counted
    span = max(sd.clip(row.name)[1], 2 * row.K) if row.K < sd.LONG_K else 2 * row.K + row.hop
    done = run_schedule(pool, span, seed=len(row.name), n_streams=1 if row.K >= sd.LONG_K else 2,
                        max_packet=max(row.K // 2 + 2 * row.hop, span // 10))
    assert done, row.name
    for x, sizes, y in done:
        with torch.no_grad(), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = row.offline(x[None])
        if row.simt:
            assert float((y - want).abs().max() / want.abs().max()) <= 1e-6, row.name
        else:
            assert torch.equal(y, want), (row.name, "pool", float((y - want).nan_to_num().abs().max()))
    if row.mod is None:
        return
    chunk = max(400, row.K // 8)
    if row.simt:
        with pytest.raises(RuntimeError, match="no fused pool route"):
            DeviceStreamPool(row.mod, S, chunk, **row.fkw)
        return
    pool = DeviceStreamPool(row.mod, S, chunk, **row.fkw)
    assert pool.T_cap == sd.device_T_cap(chunk, row.K, row.hop, row.pad, row.reflect)
    ticks = 24 if row.K >= sd.LONG_K else 40
    tr = _trace(S, chunk, ticks, len(row.name), min_end=row.K)
    xs = _inputs(S, chunk, torch.float32, ticks, len(row.name))
    want_push = row.model(S, pool.T_cap, False)[0]
    streams, rows, done = [[] for _ in range(S)], [[] for _ in range(S)], []
    for i, (ln, en, rs) in enumerate(tr):
        pool.reset(torch.as_tensor(rs).cuda())
        before = _snapshot()
        pool.push(xs[i], torch.as_tensor(ln, dtype=torch.int32).cuda(), torch.as_tensor(en).cuda())
        mine, off, other = _moved(before, row.fam)
        assert mine == want_push and not any(off) and not other, (row.name, i, mine, want_push)
        counts = pool.counts.cpu().numpy()
        tail = pool.frames.clone()
        for s in range(S):
            tail[s, :, :counts[s]] = 0
            if rs[s]:
                streams[s], rows[s] = [], []
            streams[s].append(xs[i, s, :ln[s]])
            rows[s].append(pool.frames[s:s + 1, :, :counts[s]].clone())
            if en[s]:
                done.append((torch.cat(streams[s]), _cat(rows[s])))
        assert torch.count_nonzero(tail).item() == 0, "frames past the counts are exact zeros"
    pool.check()
    for x, y in done:
        with torch.no_grad(), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = row.offline(x[None])
        assert torch.equal(y, want), (row.name, "device pool")


def _half(row, gen, B, tall_ctas):
    """bf16 / fp16 chunks equal the fp32 upcast bit for bit; the block kernel runs two MMA passes on bf16."""
    sizes = row.chunkings.get("ragged", row.chunkings["threshold"])
    x = torch.randn(B, sum(sizes), device="cuda", generator=gen)
    for dt in (torch.bfloat16, torch.float16):
        xh = x.to(dt)
        passes = 2 if dt == torch.bfloat16 else 3
        yh = _lock_step(row, xh, sizes, False, tall_ctas, passes)
        y32 = _lock_step(row, xh.float(), sizes, False, tall_ctas)
        assert torch.equal(yh, y32), (row.name, dt)


def test_stream_route_counters_skip_empty_and_refused_pushes():
    """A push of no frames counts nothing, and nor does a refused one (the CUDA-core plan under _strict)."""
    mod = build("STFT", dict(n_fft=512, hop_length=128)).cuda()
    st = StreamingTransform(mod, 1, _strict=True)
    before = _snapshot()
    st.push(torch.zeros(1, 100, device="cuda"))
    assert _moved(before, _C.ROUTES_STFT)[0] == {}
    os.environ["NNAUDIO_B200_PATH"] = "simt"
    try:
        st2 = StreamingTransform(mod, 1, _strict=True)
        before = _snapshot()
        with pytest.raises(RuntimeError, match="no fused chunk route"):
            st2.push(torch.zeros(1, 2000, device="cuda"))
        mine, off, other = _moved(before, _C.ROUTES_STFT)
        assert not mine and not any(off) and not other
    finally:
        os.environ.pop("NNAUDIO_B200_PATH")
