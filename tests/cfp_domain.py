"""Contraction list, route model, float64 stage references and shape matrix of ``Combined_Frequency_Periodicity``
/ ``CFP`` (nnaudio_b200/features/cfp.py), shared by tests/test_cfp_domain_host.py (CPU) and
tests/test_zz_gpu_cfp_domain.py (-m gpu).

One CFP forward is a chain of ``cqt1992v2_forward`` calls on the dense framed kernel (``launch_framed_tc``) or the
CUDA-core kernel: the STFT stage (a shifted ``round_up(2 (d + j), 64)``-tap bank of ``N/2 + 1`` bins, magnitude
epilogue), ``NumofLayer - 1`` cosine stages (``_RealGemm``: frames as clips of one hop ``K = round_up(N/2 + 1,
64)``, half the output rows in each bank), the frequency map on ``2B`` clips and the quefrency map.  ``calls``
lists them, ``route`` restates how each picks its kernel and what it adds to the executed-MMA-flop counter, and
``ref_stage`` contracts a call's own fp32 input and banks in float64 with the scale ``S`` its error is held to.

The end-to-end outputs pass ``pow(g)`` and ``log(relu(.) + 1e-8)``, which amplify contraction error near zero, so
each contraction is held to its own float64 reference at ``TAU[route] * S``: a bar that does not depend on that
amplification.  Each row's end-to-end bar (``bar``) is set from the split-bf16 emulation of the tensor-core routes
(``emulated_forward``); a row whose emulated error is above 1e-3 is checked stage by stage only (bar None)."""
import math

import numpy as np
import torch

import cqt1992_domain as cd
import helpers  # noqa: F401  (puts the repository on sys.path)
from nnaudio_b200 import _C
from nnaudio_b200.features.cfp import _stft_geometry

TC_BM = 128
TC_MAX_N_TILES = 128
SPLITK_MIN_K = 8192
MAX_SPLITS = 16
D, DS, S = _C.CQ1992_DENSE, _C.CQ1992_DENSE_SPLITK, _C.CQ1992_SIMT
ROUTE_NAMES = cd.ROUTE_NAMES

# |y - y64| <= TAU[route] * S + TINY over every output cell of a stage.  tests/test_cfp_domain_host.py holds each to
# at least 4x the worst ratio of the emulation (split-bf16 products summed per 64-tap block into fp32 accumulators;
# fp32 products per 16-tap block for SIMT): 2.5e-5 dense (the maps), 2.1e-6 split-K, 3e-6 SIMT.  The H100's
# accumulators lose more than that emulation on the long cosine stages, so the split-K and SIMT bars are set at
# about 4x the worst measured on an H100 SXM (700 W) instead: dense 2.7e-5 (the maps, and the 126-k-block single
# accumulator of N = 16000), split-K 1.3e-5 (N = 22050), SIMT 7.1e-5 (one fp32 accumulator over the 32832 taps of
# N = 65536, 1.5e-5 over 8064 taps).
TAU = {D: 1e-4, DS: 5e-5, S: 3e-4}
TINY = 1e-30


def _round_up(a, m):
    return -(-a // m) * m


def _ceil(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------ the calls ----
def crops(mod):
    """(n_f, n_q): the bins the two log-frequency maps read (``n_low`` clips both)."""
    N, H = mod.N, mod.N // 2 + 1
    n_low = min(int(round(N / 2)), H)
    return min(mod.HighFreqIdx, n_low), min(mod.HighQuefIdx, n_low)


def kept_frames(mod, L, drop):
    """Frames the contractions after the STFT stage see: torch.stft's count (one fewer than the kernel's
    ``L // hop + 1`` for odd N and ``L % hop == 0``), less the two edge frames when they are dropped."""
    T = (L + 2 * (mod.N // 2) - mod.N) // int(mod.hop_length) + 1
    return max(T - 2, 0) if drop else T


def calls(mod, B, L, drop):
    """Every ``cqt1992v2_forward`` call one forward of ``mod`` on (B, L) clips makes, in order: dicts with
    stage, B, L, F, K, hop, center, fmt."""
    N, W, hop = mod.N, int(mod.window_size), int(mod.hop_length)
    H = N // 2 + 1
    _, K, _ = _stft_geometry(N, W)
    out = [dict(stage="stft", B=B, L=L, F=H, K=K, hop=hop, center=True, fmt=_C.FMT_MAGNITUDE)]
    T = kept_frames(mod, L, drop)
    if T == 0:
        return out

    def gemm(stage, clips, k_in, f_out):
        Kp = _round_up(k_in, 64)
        return dict(stage=stage, B=clips, L=T * Kp, F=(f_out + 1) // 2, K=Kp, hop=Kp, center=False,
                    fmt=_C.FMT_COMPLEX)

    out += [gemm("cos", B, H, H) for _ in range(mod.NumofLayer - 1)]
    n_f, n_q = crops(mod)
    out.append(gemm("freq", 2 * B, n_f, mod.freq2logfreq_matrix.shape[0]))
    out.append(gemm("quef", B, n_q, mod.quef2logfreq_matrix.shape[0]))
    return out


def route(c, path="auto"):
    """The kernel route of one call (the bank is packed dense: no tap support) under kernel family ``path``, the
    executed MMA flops it adds, and what they were decided on."""
    F, K, hop, B, L = c["F"], c["K"], c["hop"], c["B"], c["L"]
    pad = K // 2 if c["center"] else 0
    T = (L + 2 * pad - K) // hop + 1
    bn = cd.choose_bn(F)
    n_tiles = _ceil(2 * F, bn)
    n_ph = cd.num_phases(hop)
    hop_eff = hop * n_ph
    p = dict(T=T, bn=bn, n_tiles=n_tiles, n_ph=n_ph, rows_mode=int(hop_eff % 64 == 0), ks=1, nkb=_ceil(K, 64))
    if path == "simt" or K < 16 or L + 2 * pad < K or n_tiles > TC_MAX_N_TILES:
        return dict(p, route=S, flops=0.0)
    _, ranges = cd.dense_ranges(None, F, K)
    min_range = min(hi - lo for lo, hi in ranges)
    ks = min(_ceil(min_range, 64), MAX_SPLITS, min_range) if K >= SPLITK_MIN_K else 1
    launched = min(n_ph, T)
    m_tiles = _ceil(B * _ceil(L + 2 * pad, hop_eff), TC_BM)
    kcols = sum((hi - lo) * 64 * bn for lo, hi in ranges)
    return dict(p, route=DS if ks > 1 else D, ks=ks, launched=launched,
                flops=6.0 * launched * m_tiles * TC_BM * kcols)


def plan(mod, B, L, drop, path="auto"):
    """[(call, route dict)] of one forward."""
    return [(c, route(c, path)) for c in calls(mod, B, L, drop)]


def route_totals(steps):
    """({route: calls}, summed executed flops) of a plan."""
    counts = {}
    for _, r in steps:
        counts[r["route"]] = counts.get(r["route"], 0) + 1
    return counts, sum(r["flops"] for _, r in steps)


# --------------------------------------------------------------------------------------- references ----
def frames64(x, K, hop, center):
    """(B, T, K) float64 frames of (B, L) ``x`` after ``K // 2`` zeros either side (center) or none."""
    x = torch.as_tensor(x).double()
    if center:
        x = torch.nn.functional.pad(x, (K // 2, K // 2))
    return x.unfold(1, K, hop)


def ref_stage(x, w_re, w_im, hop, center, fmt, chunk=4096):
    """Float64 (y64, S) of one call: ``y64`` the kernel's output format of (frames . w_re, -frames . w_im)
    ((B, F, T) magnitude or (B, F, T, 2) complex), ``S = |A| . |W_re| + |A| . |W_im|`` per (clip, bin, frame).
    Runs on the device of ``x``, ``chunk`` bins at a time."""
    A = frames64(x, w_re.shape[1], hop, center)
    absA = A.abs()
    ys, ss = [], []
    for f0 in range(0, w_re.shape[0], chunk):
        wr, wi = w_re[f0:f0 + chunk].double(), w_im[f0:f0 + chunk].double()
        re, im = A @ wr.T, -(A @ wi.T)
        ss.append((absA @ wr.abs().T + absA @ wi.abs().T).transpose(1, 2))
        y = torch.sqrt(re * re + im * im) if fmt == _C.FMT_MAGNITUDE else torch.stack((re, im), -1)
        ys.append(y.transpose(1, 2))
    return torch.cat(ys, 1), torch.cat(ss, 1)


def stage_ratio(y, y64, s):
    """max over cells of |y - y64| / (S + TINY), S broadcast over the complex components."""
    d = (y.double() - y64).abs()
    if d.dim() == s.dim() + 1:
        d = d.amax(-1)
    return float((d / (s + TINY)).max()) if d.numel() else 0.0


def _split(w):
    hi = w.float().bfloat16().double()
    return hi, (w.double() - hi).float().bfloat16().double()


def _accumulate(terms, block, ks):
    """sum_k A[..., k] w[f, k] over the (A, w) pairs of ``terms``: float64 partial sums over ``block``-tap blocks
    added one by one into ``ks`` fp32 accumulators (contiguous runs of blocks), which are then summed in fp32 --
    the rounding a long fp32 accumulator adds on top of the products."""
    K = terms[0][1].shape[1]
    nb = -(-K // block)
    per = -(-nb // ks)
    total = None
    for c0 in range(0, nb, per):
        acc = None
        for b in range(c0, min(nb, c0 + per)):
            k = slice(b * block, (b + 1) * block)
            part = sum(A[..., k] @ w[:, k].T for A, w in terms).float()
            acc = part if acc is None else acc + part
        total = acc if total is None else total + acc
    return total.double()


def emulated_stage(x, w_re, w_im, hop, center, fmt, r, ks=1):
    """What route ``r`` computes, emulated on the CPU: the three-term split-bf16 products (tools/sim_split_bf16.py)
    summed exactly per 64-tap k-block into ``ks`` fp32 accumulators (tensor-core routes), or fp32 products summed
    per 16-tap block into one fp32 accumulator (SIMT)."""
    K = w_re.shape[1]
    A = frames64(x.float().double(), K, hop, center)
    ah, al = _split(A)
    out = []
    for w in (w_re, w_im):
        if r == S:
            out.append(_accumulate([(A.float().double(), w.float().double())], 16, 1))
        else:
            wh, wl = _split(w)
            out.append(_accumulate([(ah, wh), (al, wh), (ah, wl)], 64, ks))
    re, im = out[0], -out[1]
    y = torch.sqrt(re * re + im * im) if fmt == _C.FMT_MAGNITUDE else torch.stack((re, im), -1)
    return y.transpose(1, 2).float()


def exact_banks(mod):
    """Float64 banks of the STFT and cosine stages, restated from the reference's definitions (the window
    zero-padded to N with ``(N - W) // 2`` zeros in front, frames centred by ``N // 2``; the cosine transform
    ``cos(2 pi n q / N) / sqrt(N)`` over the half vector) in the layout the kernel reads: tap ``m`` of the
    ``K``-wide frame is sample ``n = m - K // 2 + N // 2`` of the length-N frame; cosine output rows
    ``[0, Fh)`` in the real bank, rows ``[Fh, H)`` negated in the imaginary one."""
    N, W = mod.N, int(mod.window_size)
    H = N // 2 + 1
    _, K, _ = _stft_geometry(N, W)
    h = mod.h.detach().cpu().double()
    win = torch.zeros(N, dtype=torch.float64)
    left = (N - W) // 2
    win[left:left + W] = h / torch.linalg.norm(h)
    n = torch.arange(K) - K // 2 + N // 2
    ok = (n >= 0) & (n < N)
    wn = torch.where(ok, win[n.clamp(0, N - 1)], torch.zeros(()))
    k = torch.arange(H)[:, None]
    ang = (2.0 * math.pi / N) * ((k * n.clamp(0, N - 1)[None, :]) % N).double()
    stft = ((torch.cos(ang) * wn).contiguous(), (torch.sin(ang) * wn).contiguous())
    q = torch.arange(H)
    cosm = torch.cos((2.0 * math.pi / N) * ((q[:, None] * q[None, :]) % N).double()) / math.sqrt(N)
    Kc, Fh = _round_up(H, 64), (H + 1) // 2
    c_re = torch.zeros((Fh, Kc), dtype=torch.float64)
    c_im = torch.zeros((Fh, Kc), dtype=torch.float64)
    c_re[:, :H] = cosm[:Fh]
    c_im[:H - Fh, :H] = -cosm[Fh:]
    return dict(stft=stft, cos=(c_re, c_im))


def stage_of(mod, k_real, hop, center):
    """Which contraction a recorded call is: the STFT stage is the only centred one, a cosine stage has the
    cosine bank's shape with hop == K, the maps follow."""
    H = mod.N // 2 + 1
    if center:
        return "stft"
    if tuple(k_real.shape) == ((H + 1) // 2, _round_up(H, 64)) and hop == k_real.shape[1]:
        return "cos"
    return "map"


def exact_forward(mod, check_banks=True):
    """A float64 CPU stand-in for ``_C.cqt1992v2_forward`` under ``mod``'s host layer: the STFT and cosine
    stages contract with ``exact_banks`` (after checking that the module's fp32 banks round them), the maps with
    their fp32 buffers upcast (the values the oracle takes).  The output stays float64."""
    banks = exact_banks(mod)

    def forward(x, k_real, k_imag, packed, k_begin, k_end, hop, center, pad_mode, scale, scale_all, fmt, eps,
                path=None, strict_dtype=False):
        stage = stage_of(mod, k_real, hop, center)
        w_re, w_im = banks[stage] if stage != "map" else (k_real.double(), k_imag.double())
        if check_banks:
            for got, want in ((k_real, w_re), (k_imag, w_im)):
                assert got.shape == want.shape, (stage, got.shape, want.shape)
                assert float((got.double() - want).abs().max()) <= 1e-6 * max(float(want.abs().max()), 1e-30), stage
        A = frames64(x, w_re.shape[1], hop, center)
        re, im = (A @ w_re.T).transpose(1, 2), -(A @ w_im.T).transpose(1, 2)
        c = torch.stack((re, im), -1) * scale_all
        return torch.sqrt(re * re + im * im) * scale_all if fmt == _C.FMT_MAGNITUDE else c

    return forward


def emulated_forward(mod, path="auto", record=None):
    """A CPU stand-in for ``_C.cqt1992v2_forward`` that emulates the route each call takes (``route``); with
    ``record`` a list, appends (stage, route, ratio against the float64 contraction) per call."""

    def forward(x, k_real, k_imag, packed, k_begin, k_end, hop, center, pad_mode, scale, scale_all, fmt, eps,
                path_=None, strict_dtype=False):
        B, L = x.shape
        F, K = k_real.shape
        rt = route(dict(F=F, K=K, hop=hop, B=B, L=L, center=center), path)
        r = rt["route"]
        y = emulated_stage(x, k_real, k_imag, hop, center, fmt, r, rt["ks"])
        if record is not None:
            y64, s = ref_stage(x.double(), k_real, k_imag, hop, center, fmt)
            record.append((stage_of(mod, k_real, hop, center), r, stage_ratio(y, y64, s)))
        return y

    return forward


# ----------------------------------------------------------------------------------------- the inputs ----
def make_input(name, B=None, L=None):
    """The row's (B, L) float32 waveform (``B`` / ``L``: a shortened clip)."""
    row = ROWS[name]
    B = B or row[2][0]
    L = L or row[2][1]
    kind = row[3]
    rs = np.random.RandomState(sum(map(ord, name)))
    noise = rs.standard_normal((B, L))
    if kind[0] == "randn":
        x = noise
    elif kind[0] == "silence":
        x = np.zeros((B, L))
    elif kind[0] == "dc":
        x = kind[1] + noise
    elif kind[0] == "tone":  # a sine at the centre of STFT bin kind[1], plus a little noise
        fs = row[1].get("fs", 16000)
        N = int(fs / float(row[1].get("fr", 2)))
        x = np.sin(2 * np.pi * kind[1] / N * np.arange(L))[None, :] + 1e-3 * noise
    elif kind[0] == "impulse":
        x = np.zeros((B, L))
        x[:, L // 3] = 1.0
        x[:, (2 * L) // 3] = -0.5
    elif kind[0] == "amp":
        x = kind[1] * noise
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(x, dtype=np.float32)


# ------------------------------------------------------------------------------------------ the matrix ----
CLASSES = {"CFP": "CFP", "Comb": "Combined_Frequency_Periodicity"}
RN = ("randn",)
# name -> (class, constructor, (B, L), input, claims, options).  Claims: N, the STFT stage's bank width K, and the
# route of each stage kind ("stft", "cos", "freq", "quef") under path auto; kept (frames after the crop).
# Options: attrs (module attributes set after construction: cut-off indices no constructor can reach), bar (the
# end-to-end bar of Z / tfrLF / tfrLQ; None: stage-only), host (B, L) of the CPU checks when the clip is shortened,
# null (outputs that are exactly zero: a constant spectrum -- g[0] = 0, or the flat magnitude of one impulse per
# frame -- lies wholly in the frame mean, which the cepstral cut-off removes; the float64 FFT of the oracle leaves
# round-off there, so those outputs are held to zero instead).
ROWS = {
    # ---- transform size: even / odd N, fr, fs
    "default": ("CFP", {}, (2, 8000), RN, dict(N=8000, K=2112, stft=D, cos=D), {}),
    "comb_default": ("Comb", {}, (2, 8000), RN, dict(N=8000, stft=D, cos=D, kept=24), {}),
    "fs8000_fr2": ("Comb", dict(fs=8000), (2, 8000), RN, dict(N=4000, stft=D, cos=D), {}),
    "odd_n_fr3": ("Comb", dict(fr=3), (2, 8000), RN, dict(N=5333, stft=D, cos=D), {}),
    "fr4": ("Comb", dict(fr=4), (2, 8000), RN, dict(N=4000, stft=D, cos=D), {}),
    "fr8": ("Comb", dict(fr=8, window_size=1025), (2, 8000), RN, dict(N=2000, stft=D, cos=D), {}),
    "fs22050_fr2_odd": ("Comb", dict(fs=22050, hop_length=441), (2, 11025), RN, dict(N=11025, cos=D), {}),
    "n16000_cos_k8064": ("Comb", dict(fr=1), (2, 8000), RN, dict(N=16000, stft=D, cos=D, cos_K=8064), {}),
    "n22050_cos_splitk": ("Comb", dict(fs=22050, fr=1, hop_length=441), (1, 8820), RN,
                          dict(N=22050, stft=D, cos=DS, cos_ks=3), {}),
    "n44100_stft_simt": ("Comb", dict(fs=44100, fr=1, hop_length=441), (1, 2205), RN,
                         dict(N=44100, stft=S, cos=DS, cos_ks=6), dict(bar=None)),
    "n65536_cos_simt": ("Comb", dict(fs=65536, fr=1, hop_length=1024), (1, 3072), RN,
                        dict(N=65536, stft=S, cos=S), dict(bar=None)),
    # ---- window
    "window_eq_n_even": ("Comb", dict(fr=4, window_size=4000), (2, 8000), RN, dict(N=4000, K=4032), {}),
    "window_eq_n_odd": ("Comb", dict(fr=3, window_size=5333), (2, 8000), RN, dict(N=5333, K=5376, j=22), {}),
    "window_tiny_65": ("Comb", dict(window_size=65), (2, 8000), RN, dict(N=8000, K=128), dict(bar=None)),
    "window_just_under_n": ("Comb", dict(window_size=7999), (2, 8000), RN, dict(K=8000, stft=D), {}),
    "window_4097_k4160": ("Comb", dict(window_size=4097), (2, 8000), RN, dict(K=4160, stft=D), {}),
    "stft_splitk_12001": ("Comb", dict(fr=1, window_size=12001), (1, 8000), RN, dict(K=12032, stft=DS, stft_ks=3),
                          {}),
    # ---- hop
    "hop64_rows": ("Comb", dict(hop_length=64), (2, 4000), RN, dict(stft_n_ph=1, stft_rows_mode=1), {}),
    "hop100_2ph": ("Comb", dict(hop_length=100), (2, 6000), RN, dict(stft_n_ph=2), {}),
    "hop250_4ph": ("Comb", dict(hop_length=250), (2, 8000), RN, dict(stft_n_ph=4), {}),
    "hop441_8ph": ("Comb", dict(hop_length=441), (2, 8000), RN, dict(stft_n_ph=8), {}),
    "hop_gt_window": ("Comb", dict(window_size=1025, hop_length=1500), (2, 12000), RN, dict(kept=7), {}),
    "hop_gt_n": ("CFP", dict(fs=8000, hop_length=5000), (2, 16000), RN, dict(N=4000, kept=4), {}),
    # ---- length and batch
    "cfp_l_lt_hop": ("CFP", {}, (3, 200), RN, dict(kept=1, stft_T=1), {}),
    "comb_T1": ("Comb", {}, (2, 200), RN, dict(kept=0), {}),
    "comb_T2": ("Comb", {}, (2, 500), RN, dict(kept=0), {}),
    "comb_T3": ("Comb", {}, (2, 700), RN, dict(kept=1), {}),
    "b1": ("CFP", {}, (1, 16000), RN, dict(kept=51), {}),
    "b40_m_tiles": ("Comb", {}, (40, 8000), RN, dict(kept=24, cos_m_tiles=8), dict(host=(4, 8000))),
    # ---- layers
    "g2": ("Comb", dict(g=[0.24, 0.6]), (2, 8000), RN, dict(layers=2), {}),
    "g4": ("Comb", dict(g=[0.24, 0.6, 1, 0.5]), (2, 8000), RN, dict(layers=4), {}),
    "g5": ("Comb", dict(g=[0.24, 0.6, 1, 0.5, 0.8]), (2, 8000), RN, dict(layers=5), dict(bar=2e-3)),
    "g_log_ceps": ("Comb", dict(g=[0.24, 0, 1]), (2, 8000), RN, {}, dict(bar=None)),
    "g_log_spec": ("Comb", dict(g=[0.24, 0.6, 1, 0]), (2, 8000), RN, {}, dict(bar=5e-4)),
    "g0_zero": ("Comb", dict(g=[0, 0.6, 1]), (2, 8000), RN, {}, dict(null=(0, 2, 3))),
    # ---- cut-offs and crops
    "tc_idx_0": ("Comb", {}, (2, 8000), RN, {}, dict(attrs=dict(tc_idx=0))),
    "fc_idx_0": ("Comb", {}, (2, 8000), RN, {}, dict(attrs=dict(fc_idx=0))),
    "cut_past_half": ("Comb", dict(g=[0.24, 0.6, 1, 0.5]), (2, 8000), RN, {}, dict(attrs=dict(tc_idx=4003))),
    "high_freq_clipped": ("Comb", dict(fs=8000, tc=1 / 5000, NumPerOct=1), (2, 8000), RN,
                          dict(N=4000, n_f=2000), {}),
    # ---- input
    "silence": ("Comb", {}, (2, 8000), ("silence",), {}, {}),
    "dc_offset_1000x": ("Comb", {}, (2, 8000), ("dc", 1000.0), {}, dict(bar=None)),
    "tone_bin_centre": ("Comb", {}, (2, 8000), ("tone", 441), {}, dict(bar=None)),
    "impulse": ("Comb", {}, (2, 8000), ("impulse",), {}, dict(bar=None, null=(0, 2, 3))),
    "amp_1e-4": ("Comb", {}, (2, 8000), ("amp", 1e-4), {}, {}),
    "amp_1e4": ("Comb", {}, (2, 8000), ("amp", 1e4), {}, {}),
}
DEFAULT_OPTS = dict(attrs={}, bar=3e-4, host=None, null=())


def row_options(name):
    return dict(DEFAULT_OPTS, **ROWS[name][5])


def build_row(name):
    cls, ctor = ROWS[name][:2]
    mod = helpers.build(CLASSES[cls], ctor)
    for k, v in row_options(name)["attrs"].items():
        setattr(mod, k, v)
    return mod


def drops(name):
    return ROWS[name][0] == "Comb"


def run_oracle(mod, x, drop):
    return helpers.oracle.cfp(np.asarray(x, dtype=np.float64), mod.h.cpu().numpy(),
                              mod.freq2logfreq_matrix.cpu().numpy(), mod.quef2logfreq_matrix.cpu().numpy(), mod.N,
                              mod.hop_length, mod.g, mod.tc_idx, mod.fc_idx, mod.HighFreqIdx, mod.HighQuefIdx,
                              drop_edge_frames=drop)
