"""Shape matrix, chunkings and per-push launch model of the streamed calls: ``StreamingTransform`` / ``StreamPool`` /
``DeviceStreamPool`` (STFT, MelSpectrogram, Gammatonegram, MFCC, CQT1992v2), ``StreamingPyramid`` / ``PyramidPool``
/ ``DevicePyramidPool`` and ``StreamingInverse``.  Shared by tests/test_stream_domain_host.py (CPU) and
tests/test_zz_gpu_stream_domain*.py (-m gpu).

The rows are the offline domain matrices, taken by name (dense_domain, cqt1992_domain, block_domain's module
shapes, pyramid_domain, ola_domain's inverse STFT), plus three stream-only edges.  A push runs the offline plan on
its virtual clip: A rows of (T_max - 1) hop + K samples with no padding (a device pool: every slot, T_cap frames), so
its routes and executed flops are the offline model's on that geometry (``stft_push``, ``cq1992_push``,
``pyramid_push``, ``istft_push`` call the domain modules' models with it).

Rows whose class has a ``direct:`` prefix (n_fft >= 8192: a module would design gigabytes of float64 on the host)
stream through a ``StreamingTransform`` made without ``__init__`` (``direct_stream``): its counters, readiness rule,
push, flush and concat route are the class's own, only the offline arguments come from the device-built basis.  A
test-local state object would restate those rules, and a module subclass would still have to fake the float64
design; the bypass keeps the code under test the code users run."""
import numpy as np
import torch

import block_domain as bd
import cqt1992_domain as cd
import dense_domain as dd
import ola_domain as od
import pyramid_domain as pd
from nnaudio_b200 import _C
from nnaudio_b200.streaming import StreamingInverse, StreamingTransform, _ready_frames

LONG_K = 16384  # K >= LONG_K: threshold cuts only

# ----------------------------------------------------------------------------------------------- the matrix ----
# STFT family: rows in dense_domain's layout (class, constructor, (B, L), claims, options); CQT1992v2: rows in
# cqt1992_domain's layout (class, constructor, B, L, (F, K, hop), route, claims, options).  Every row carries its edge.
STFT_ROWS = {f"dense:{k}": v for k, v in dd.ROWS.items()}
for _n, _h, _B, _L in bd.STFT_SHAPES:
    STFT_ROWS[f"block:{_n}_{_h}"] = ("STFT", dict(n_fft=_n, hop_length=_h), (_B, _L), {}, {})
for _n, _h in bd.PAD_SHAPES:
    _B, _L = next((b, ln) for n, h, b, ln in bd.STFT_SHAPES if (n, h) == (_n, _h))
    STFT_ROWS[f"block:{_n}_{_h}_no_center"] = ("STFT", dict(n_fft=_n, hop_length=_h, center=False), (_B, _L), {}, {})
    STFT_ROWS[f"block:{_n}_{_h}_constant"] = ("STFT", dict(n_fft=_n, hop_length=_h, pad_mode="constant"),
                                              (_B, _L), {}, {})
STFT_ROWS["stream:hop_over_nfft_dense"] = ("STFT", dict(n_fft=256, hop_length=384, window="hamming"),
                                           (2, 384 * 30 + 101), dict(routes={_C.STFT_DENSE: 1}, n_ph=1), {})
STFT_ROWS["stream:half_hop_reflect"] = ("STFT", dict(n_fft=512, hop_length=256), (2, 256 * 40 + 3),
                                        dict(routes={_C.STFT_BLOCK: 1}), {})
CQ_ROWS = {f"cqt:{k}": v for k, v in cd.ROWS.items()}
CQ_ROWS["stream:cqt_narrower_than_hop"] = ("CQT1992v2", dict(sr=16000, fmin=2000, n_bins=24, hop_length=512), 2,
                                           16000, (24, 256, 512), _C.CQ1992_DENSE, {}, {})
EDGES = {
    "stream:hop_over_nfft_dense": "hop 384 > n_fft 256: frames skip samples, the ring keeps no overlap",
    "stream:half_hop_reflect": "hop = n_fft / 2, reflect: the right mirror of a push reads pad + 1 samples back",
    "stream:cqt_narrower_than_hop": "kernel_width 256 < hop 512 on the dense kernel",
}
for _k in STFT_ROWS:
    EDGES.setdefault(_k, "dense_domain row" if _k.startswith("dense:") else "block_domain module shape")
for _k in CQ_ROWS:
    EDGES.setdefault(_k, "cqt1992_domain row")
FORWARD = sorted(STFT_ROWS) + sorted(CQ_ROWS)
PYRAMID = sorted(pd.ROWS)
INVERSE = sorted(od.ISTFT_ROWS)


def is_stft(name):
    return name in STFT_ROWS


def base_class(name):
    row = STFT_ROWS.get(name) or CQ_ROWS[name]
    return row[0].split(":")[-1]


def is_direct(name):
    return is_stft(name) and STFT_ROWS[name][0].startswith("direct:")


def options(name):
    if is_stft(name):
        return dict(dd.DEFAULT_OPTS, **STFT_ROWS[name][4])
    return dict(cd.DEFAULT_OPTS, **CQ_ROWS[name][7])


def constructor(name):
    """The row's constructor; MFCC streams only without the per-clip top_db floor."""
    row = STFT_ROWS.get(name) or CQ_ROWS[name]
    ctor = dict(row[1])
    if base_class(name) == "MFCC":
        ctor["top_db"] = None
    return ctor


def clip(name):
    """(B, L) of the row."""
    if is_stft(name):
        return STFT_ROWS[name][2]
    return CQ_ROWS[name][2], CQ_ROWS[name][3]


def geometry(name, kernel_width=None):
    """(K, hop, pad, reflect) of a row's stream (a CQT row: K is the module's kernel width)."""
    if is_stft(name):
        K, _, hop, center, pad_mode, _, _ = dd.row_geometry(name, STFT_ROWS[name])
    else:
        ctor = CQ_ROWS[name][1]
        K, hop = kernel_width or CQ_ROWS[name][4][1], CQ_ROWS[name][4][2]
        center, pad_mode = ctor.get("center", True), ctor.get("pad_mode", "reflect")
    pad = K // 2 if center else 0
    return K, hop, pad, pad > 0 and pad_mode == "reflect"


def bank(name):
    """The (n_fb, F) float64 filterbank of a dense_domain row (None for every other row)."""
    return dd.bank(name.split(":", 1)[1]) if name.startswith("dense:") else None


def pyramid_geometry(mod):
    """(F, widths, top-level hop, early factor, generation) of a pyramid module's streams: generation 2 without early
    downsampling when every FIR-source bank is 256 wide (StreamingPyramid's rule), else 1."""
    F, widths = pd.bank_shapes(mod)
    e = pd.early_factor(mod)
    gen = 2 if e == 1 and all(w // 2 == 128 for w in widths[:-1]) else 1
    return F, widths, pd.levels(mod, pd.valid_length(mod, 1 << 16))[0].hop, e, gen


def pyramid_streams(mod):
    """StreamingPyramid takes the module: the octaves frame at one rate (hop a multiple of 2^(n_octaves - 1))."""
    _, widths, hop, _, _ = pyramid_geometry(mod)
    return hop % (1 << (len(widths) - 1)) == 0


def auto_simt(name):
    """The row's plan is the CUDA-core kernel (forced, or the auto plan's): no fused chunk route."""
    if is_stft(name):
        return _C.STFT_SIMT in STFT_ROWS[name][3].get("routes", {}) or options(name)["path"] == "simt"
    return CQ_ROWS[name][5] == _C.CQ1992_SIMT


# ------------------------------------------------------------------------------------------- chunkings ----
def flush_frames(total, K, hop, pad):
    return max(0, (total + 2 * pad - K) // hop + 1)


def simulate(sizes, K, hop, pad, reflect):
    """Frames each push of ``sizes`` returns, then the flush's: the readiness rule of StreamingTransform."""
    total = frames = 0
    out = []
    for n in sizes:
        total += n
        t = _ready_frames(total, K, hop, pad, reflect)
        out.append(t - frames)
        frames = t
    out.append(flush_frames(total, K, hop, pad) - frames)
    return out


def _fill(sizes, L, step):
    """``sizes`` then pushes of ``step`` up to L samples in all."""
    sizes = list(sizes)
    while sum(sizes) < L:
        sizes.append(min(step, L - sum(sizes)))
    return sizes


def chunkings(K, hop, pad, reflect, L, n_ph=1, seed=0):
    """name -> push sizes of one stream (its length is their sum; a flush follows), derived from the readiness
    rule.  "threshold": a push ending at K - pad - 1 samples, the next at K - pad, then one more sample (the reflect
    threshold pad + 1 for an even K), a zero-length push, a push longer than K, pushes of ~0.6 K past two ring wraps,
    and a length whose flush returns no new frame where the framing has one.  "pad_plus_one" (reflect): a stream of
    pad + 1 samples.  "short" (centred): K - 1 samples, frames from the padding only.  "phases" (n_ph > 1): pushes
    returning more, and fewer, frames than the dense kernel's frame phases.  "ragged": seeded cuts.  Rows with
    K >= LONG_K keep the threshold and pad + 1 streams only."""
    need = K - pad
    head = [need - 1, 1, 1, 0, K + 2 * hop + 1]
    L0 = max(L, 2 * K + need + 3 * hop)
    # the stream length: the first from L0 whose flush returns nothing new, where one is near
    L_thr = next((t for t in range(L0, L0 + K + 2 * hop)
                  if flush_frames(t, K, hop, pad) == _ready_frames(t, K, hop, pad, reflect)), L0)
    out = {"threshold": _fill(head, L_thr, 3 * K // 5 + 1)}
    if reflect:
        out["pad_plus_one"] = [pad, 1]
    if K >= LONG_K:
        return out
    if pad > 0:
        out["short"] = [K // 3, K - 1 - K // 3]
    if n_ph > 1:
        out["phases"] = _fill([need + hop * (n_ph + 2), hop, 0, hop, hop * (n_ph + 3) + 1], max(L, need + hop * 40),
                              hop * (n_ph - 1))
    rng = np.random.default_rng(seed)
    sizes = []
    while sum(sizes) < L:
        sizes.append(int(min(rng.integers(0, K + 2 * hop + 2), L - sum(sizes))))
    out["ragged"] = sizes
    return out


def row_chunkings(name, kernel_width=None):
    K, hop, pad, reflect = geometry(name, kernel_width)
    B, L = clip(name)
    n_ph = dd.num_phases(hop)
    return chunkings(K, hop, pad, reflect, L, n_ph, seed=len(name))


def properties(sizes, K, hop, pad, reflect, n_ph=1):
    """What one chunking reaches (the claims of ``chunkings``)."""
    got = simulate(sizes, K, hop, pad, reflect)
    totals = np.cumsum(sizes).tolist()
    pushes = got[:-1]
    p = set()
    need = K - pad
    for i in range(1, len(totals)):
        if totals[i - 1] == need - 1 and totals[i] == need:
            p.add("threshold")
        if pushes[i - 1] > 0 and pushes[i] == 0:
            p.add("zero_after_frames")
    if reflect and sum(sizes) == pad + 1:
        p.add("pad_plus_one")
    if sum(sizes) < K and sum(got) > 0:
        p.add("shorter_than_K")
    if any(n > K for n in sizes):
        p.add("longer_than_K")
    if sum(sizes) >= 2 * K:
        p.add("two_wraps")
    if 0 in sizes:
        p.add("zero_length")
    if got[-1] == 0:
        p.add("empty_flush")
    if any(0 < t < n_ph for t in pushes):
        p.add("fewer_than_phases")
    if any(t > n_ph for t in pushes) and n_ph > 1:
        p.add("more_than_phases")
    return p


def empty_flush_possible(K, hop, pad, reflect, L):
    return any(flush_frames(t, K, hop, pad) == _ready_frames(t, K, hop, pad, reflect)
               for t in range(L, L + K + 2 * hop))


# ---------------------------------------------------------------------------------------- push model ----
def virtual_clip(T_max, K, hop):
    return (T_max - 1) * hop + K


def stft_push(name, A, T_max, fb=None, passes=3):
    """dense_domain.plan of a push: A rows of the virtual clip, no padding."""
    K, F, hop, _, _, block, _ = dd.row_geometry(name, STFT_ROWS[name])
    return dd.plan(K, F, hop, A, virtual_clip(T_max, K, hop), False, block, options(name)["path"], fb, passes)


class Uncentred:
    """A CQT module seen with center=False: the geometry cqt1992_domain.plan reads for a push."""
    center = False

    def __init__(self, mod):
        self._mod = mod

    def __getattr__(self, k):
        return getattr(self._mod, k)


def cq1992_push(mod, A, T_max, balance=True, tall_ctas=None):
    """cqt1992_domain.plan of a push: A rows of the virtual clip, no padding."""
    K, hop = int(mod.kernel_width), int(mod.hop_length)
    return cd.plan(Uncentred(mod), A, virtual_clip(T_max, K, hop), "auto", tall_ctas=tall_ctas, balance=balance)


def pyramid_push(F, widths, hop, rows, gen2, fir_stages):
    """Stream counter deltas of one pyramid push that returns frames (F filters per octave, bank ``widths``, top
    level ``hop``): the plan once, each octave on ``rows`` rows (generation 2: the octave kernel when octave_tc_ok,
    else the dense kernel on the level planes when hop % 8 == 0; otherwise the dense kernel from the fp32 rows), and
    one FIR route per stage that launched (``fir_stages``)."""
    r = {_C.PYR_PLAN_GEN2 if gen2 else _C.PYR_PLAN_GEN1: 1}
    for i, w in enumerate(widths):
        h = hop >> i
        k = (_C.PYR_OCT_KERNEL if gen2 and pd.presplit(h) and pd.octave_tc_ok(F, w, h, rows)
             else _C.PYR_OCT_DENSE_PLANES if gen2 and pd.presplit(h) else _C.PYR_OCT_DENSE_FP32)
        r[k] = r.get(k, 0) + 1
    if fir_stages:
        r[_C.PYR_FIR_BANDED if gen2 else _C.PYR_FIR_DENSE] = fir_stages
    return r


def fir_stages_launched(plan_rows):
    """FIR stages a pyramid push launches: the signals (all but the last) that some lane advances (first FIR row
    >= 0 in ``_C.cqt_pyramid_chunk_plan`` / ``cqt_pyramid_pool_plan``)."""
    return sum(any(sig[s][5] >= 0 for sig in plan_rows) for s in range(len(plan_rows[0]) - 1))


def istft_push(rows, T_max, n_fft, f_in):
    """Executed flops of an inverse push: the overlap-add GEMM of rows x T_max frames (its K chunks included)."""
    return od.ola_exec_flops(*od.istft_operands(rows, T_max, n_fft, f_in))


def device_T_cap(chunk, K, hop, pad, reflect):
    """The most frames one push of at most ``chunk`` samples returns, an end included, by the readiness rule: over
    every position R the stream can be at (the framing repeats every hop samples past K + 2 chunk)."""
    R = np.arange(0, K + 2 * chunk + 2 * hop)
    ready = np.array([_ready_frames(int(r), K, hop, pad, reflect) for r in R])
    end = np.maximum(0, (R + chunk + 2 * pad - K) // hop + 1)
    return int((end - ready).max())


# ------------------------------------------------------------------------------------ direct-basis streams ----
def direct_stream(name, kw, batch, device):
    """A StreamingTransform of a ``direct:`` row on the offline arguments ``kw`` of ``_C.<name>`` (the device-built
    basis), made without __init__ (see the module docstring)."""
    cls = base_class(name)
    call = "stft_forward" if cls == "STFT" else "stft_filterbank_forward"
    K, hop, pad, reflect = geometry(name)
    st = StreamingTransform.__new__(StreamingTransform)
    st.module, st.batch, st._strict = None, batch, False
    st._args = lambda: (call, kw)
    st._check_length = lambda n: None
    st.K, st.hop, st.pad, st._reflect = K, hop, pad, reflect
    st.ring = torch.empty((batch, K), dtype=torch.float32, device=device)
    st.reset()
    return st


def direct_inverse(packed, window, n_fft, hop, center, onesided, batch, device):
    """A StreamingInverse on a device-built packed basis (n_fft >= 8192), made without __init__ as
    ``direct_stream``."""
    si = StreamingInverse.__new__(StreamingInverse)
    si.module, si.batch, si.onesided = None, batch, onesided
    si.n_fft, si.hop, si.center = n_fft, hop, center
    si.f_in = n_fft // 2 + 1 if onesided else n_fft
    si._args = lambda: (None, None, packed, window)
    si.offset = n_fft // 2 if center else 0
    si.state = torch.empty((batch, n_fft), dtype=torch.float32, device=device)
    si.reset()
    return si

