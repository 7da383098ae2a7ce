"""Float64 stage references, launch model and shape matrix of ``Griffin_Lim``, shared by
tests/test_griffin_domain_host.py (CPU) and tests/test_zz_gpu_griffin_domain.py (-m gpu).

One Griffin-Lim iteration is three stages: the inverse STFT (the overlap-add GEMM of csrc/tc_kernels.cu), the forward
STFT with Complex output (the block-partial, dense or CUDA-core kernel ``dense_domain.plan`` picks) and the
elementwise phase update in torch between them.  The whole loop cannot be compared tightly with anything: the update
divides by |angles|, which amplifies rounding wherever |angles| ~ 0 and feeds it to the next iteration.  So each stage
is held to float64 on the float32 inputs the module itself recorded for it, and no drift accumulates:

- ``ref_inverse`` / ``ref_forward`` are tests/ola_domain.py's and tests/dense_domain.py's references of the two
  transforms, the forward on the module's own ``wcos`` / ``wsin``;
- ``ref_update`` is the momentum step and the phase renormalisation, and ``glue_bound`` is what float32 rounding may
  move it by, cell by cell;
- ``ref_loop`` composes the three; tests/test_griffin_domain_host.py holds it to ``oracle.griffin_lim``.

``call_model`` restates which forward route each iteration takes and the executed MMA flops a whole call adds, so a
test that reads the counters proves which kernels ran.  The shape matrix ``ROWS`` names the edge each row is there
for."""
import numpy as np

import dense_domain as dd
import ola_domain as od
from nnaudio_b200 import _C

U = 2.0 ** -24        # unit roundoff of float32
EPS = 1e-16           # the update's guard against |angles| = 0 (griffin_lim.py:136)
MAX_BATCH = 65535     # clips per C call: larger batches run in chunks


# ------------------------------------------------------------------------------------------ references ----
def cplx(a):
    """(..., 2) real pairs -> complex128."""
    a = np.asarray(a, dtype=np.float64)
    return a[..., 0] + 1j * a[..., 1]


def ref_inverse(X, win, hop):
    """(B, F, T) complex one-sided spectrogram -> (B, hop (T - 1)) float64 waveform: the centred inverse STFT with
    the window ``win`` (``od.ref_istft``: the window sum-square divides only where it exceeds 1e-10)."""
    X = np.asarray(X)
    return od.ref_istft(np.stack((X.real, X.imag), -1), win, hop, True, True, None)[0]


def ref_forward(y, wcos, wsin, hop, pad_mode):
    """(B, L) waveform -> (B, F, T) complex128: the centred STFT of the bases ``wcos`` / ``wsin`` upcast to float64
    (``dd.ref_stft``), so the module's fp32 bases are the reference's and their rounding is not kernel error."""
    return dd.ref_stft(y, wcos, wsin, hop, True, pad_mode)


def ref_update(r, p, momentum):
    """The phase update of one iteration: a = r - m / (1 + m) p, then a / (|a| + 1e-16); complex in and out."""
    a = np.asarray(r, dtype=np.complex128) - (momentum / (1.0 + momentum)) * np.asarray(p, dtype=np.complex128)
    return a / (np.abs(a) + EPS)


def ref_initial(phase):
    """The first inverse's phase factors cos 2 pi phase + i sin 2 pi phase of the float32 phase."""
    ph = 2.0 * np.pi * np.asarray(phase, dtype=np.float32).astype(np.float64)
    return np.cos(ph) + 1j * np.sin(ph)


def ref_loop(S, phase, hop, win, wcos, wsin, n_iter, momentum, pad_mode):
    """The whole loop in float64 from the three stage references: ``n_iter`` inverse / forward / update rounds,
    then a last inverse.

    It differs from ``oracle.griffin_lim`` (the reference source restated) in one place: the oracle divides the
    overlap-add by the window sum-square unconditionally, as ``torch.istft`` does, while the library and
    ``od.ref_istft`` divide only where it exceeds 1e-10.  Where the window sum-square is zero inside the output -- a
    Hann window at hop == n_fft -- the oracle returns non-finite samples and this reference keeps the undivided sum.
    Everywhere the window sum-square is positive the two agree to float64 rounding."""
    S = np.asarray(S, dtype=np.float32).astype(np.float64)
    angles = ref_initial(phase)
    rebuilt = np.zeros_like(angles)
    for _ in range(n_iter):
        tprev = rebuilt
        rebuilt = ref_forward(ref_inverse(S * angles, win, hop), wcos, wsin, hop, pad_mode)
        angles = ref_update(rebuilt, tprev, momentum)
    return ref_inverse(S * angles, win, hop)


def glue_bound(r, p, momentum, S):
    """Elementwise bound (B, F, T), per real component, on |S * angles - S * ref_update(r, p, m)| when ``angles``
    is the update evaluated in float32 torch from the float32 ``r`` (this iteration's forward output) and ``p`` (the
    previous one), as ``Griffin_Lim.forward`` does, and S * angles is rounded to float32.

    Derivation (u = 2^-24, every float32 operation correctly rounded, d = m / (1 + m) rounded to float32 when it
    scales the tensor, a = r - d p exact):
    - t = d p rounds twice: t = d p (1 + th), |th| <= 2.01 u; a^ = (r - t)(1 + de) differs from a by at most
      u |a_c| + 2.01 u d |p_c| per component, so |a^ - a| <= 1.5 u (|r| + 4 d |p|) =: E as a vector (the 1.5 covers
      the step from two components to their norm);
    - |a^| from two squares, a sum and a square root carries 2.5 u, adding 1e-16 one more u, the division one more u:
      those move a unit-modulus quotient by at most 4.6 u per component;
    - x -> x / |x| moves by at most 2 |x - y| / |y|, so a^ / |a^| is within 2 E / (|a| + 1e-16) of a / (|a| + 1e-16);
    - multiplying by S rounds once more, by at most u S.
    So the bound is S u (3 (|r| + 4 d |p|) / (|a| + 1e-16) + 6).  It grows without limit where |a| -> 0; those cells
    are not masked, because there the float32 update is as uncertain as the bound says."""
    r = np.asarray(r, dtype=np.complex128)
    p = np.asarray(p, dtype=np.complex128)
    d = momentum / (1.0 + momentum)
    a = np.abs(r - d * p)
    S = np.asarray(S, dtype=np.float32).astype(np.float64)
    return S * U * (3.0 * (np.abs(r) + 4.0 * d * np.abs(p)) / (a + EPS) + 6.0)


def initial_bound(phase, S):
    """Elementwise bound on |S * cos(2 pi phase) - float32 torch's value| (and the same for sin): 2 pi phase
    rounds twice (2.01 u |2 pi phase|), the float32 cos / sin is within 2 ulp (4 u), the product with S one u."""
    th = np.abs(2.0 * np.pi * np.asarray(phase, dtype=np.float32).astype(np.float64))
    S = np.asarray(S, dtype=np.float32).astype(np.float64)
    return S * U * (2.01 * th + 5.0)


def ratio(diff, bound):
    """Largest |diff| / bound, with 0 / 0 = 0 and anything over a zero bound infinite."""
    diff = np.abs(diff)
    bound = np.asarray(bound, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(diff == 0, 0.0, diff / bound)
    return float(q.max()) if q.size else 0.0


# ---------------------------------------------------------------------------------------------- recorder ----
class Recorder:
    """Records every stage call of a ``Griffin_Lim`` module: within ``with Recorder(mod) as rec:`` the module's
    ``_inverse`` and ``_stft.forward`` are wrapped (instance attributes), and ``rec.calls`` collects
    ("inverse" | "forward", float32 input, float32 output) as host copies, in call order."""

    def __init__(self, mod):
        self.mod = mod
        self.calls = []

    def __enter__(self):
        inv, fwd = self.mod._inverse, self.mod._stft.forward

        def inverse(spec):
            out = inv(spec)
            self.calls.append(("inverse", spec.detach().cpu(), out.detach().cpu()))
            return out

        def forward(x, output_format=None):
            out = fwd(x, output_format=output_format)
            self.calls.append(("forward", x.detach().cpu(), out.detach().cpu()))
            return out

        self.mod._inverse = inverse
        self.mod._stft.forward = forward
        return self

    def __exit__(self, *exc):
        del self.mod._inverse
        del self.mod._stft.forward
        return False

    def kinds(self):
        return [k for k, _, _ in self.calls]

    def inverses(self):
        return [(i, o) for k, i, o in self.calls if k == "inverse"]

    def forwards(self):
        return [(i, o) for k, i, o in self.calls if k == "forward"]


def call_order(n_iter):
    return ["inverse", "forward"] * n_iter + ["inverse"]


# ------------------------------------------------------------------------------------------ shape matrix ----
# name -> n_fft, hop, T (frames of S), B, n_iter, momentum, window, win_length, pad_mode, route (the forward's
# STFT_* route) and edge.  T is the spectrogram's frames; the clips the loop rebuilds have hop (T - 1) samples.
BLK, DENSE = _C.STFT_BLOCK, _C.STFT_DENSE
ROWS = {}


def _row(name, n_fft, hop, route, edge, T=40, B=2, n_iter=4, momentum=0.99, window="hann", win_length=None,
         pad_mode="reflect"):
    assert name not in ROWS
    ROWS[name] = dict(n_fft=n_fft, hop=hop, T=T, B=B, n_iter=n_iter, momentum=momentum, window=window,
                      win_length=win_length, pad_mode=pad_mode, route=route, edge=edge)


# ---- block-partial forward
_row("block1_256_64", 256, 64, BLK, "one-phase block kernel, R = 4 (the n_fft 256 configuration of "
     "test_griffin_lim.py, kept as the anchor)", n_iter=6)
_row("block1_384_192", 384, 192, BLK, "one-phase block kernel, R = 2, n_fft not a power of two; an overlap-add of "
     "two frames per sample, so deterministic", T=30)
_row("block4_512_128", 512, 128, BLK, "four-phase block kernel, R = 4", T=30)
_row("block4_1024_512", 1024, 512, BLK, "four-phase block kernel, R = 2: deterministic four-phase row", T=20)
_row("block4_2048_512", 2048, 512, BLK, "four-phase block kernel at n_fft 2048", T=16, n_iter=3)
_row("block4_8192_2048", 8192, 2048, BLK, "four-phase block kernel with 11 N tiles; three overlap-add K chunks",
     T=6, B=1, n_iter=2)
# ---- dense forward
_row("dense_hamming_512_128", 512, 128, DENSE, "non-Hann window (the hamming configuration of "
     "test_griffin_lim.py): dense kernel", T=30, window="hamming", win_length=400, momentum=0.5)
_row("dense_400_160", 400, 160, DENSE, "hop % 64 != 0: dense kernel, one frame phase", T=30)
_row("dense_1000_250", 1000, 250, DENSE, "dense kernel over four frame phases, partial fourth overlap-add N tile",
     T=20)
_row("dense_512_160_wl400", 512, 160, DENSE, "Hann window cut to win_length 400: not the block layout", T=30,
     win_length=400)
# ---- padding and length edges
_row("constant_T2", 256, 64, BLK, "constant padding at the shortest T that runs (one hop of samples)", T=2,
     pad_mode="constant")
_row("reflect_T4", 256, 64, BLK, "reflect padding at the shortest T that runs: hop (T - 1) = 192 > n_fft / 2",
     T=4)
# ---- loop edges
_row("momentum0", 256, 64, BLK, "momentum 0: the update is a pure projection", momentum=0.0)
_row("n_iter0", 256, 64, BLK, "n_iter 0: one inverse of the initial phase, no forward", n_iter=0)
_row("n_iter1", 512, 128, BLK, "n_iter 1: the update reads the zero tprev only", T=20, n_iter=1)
_row("mtile_B37_T5", 256, 64, BLK, "B T = 185 rows straddle 128-row M tiles, clips of 256 samples", T=5, B=37)
# ---- batches past one C call
_row("b65536_128_32", 128, 32, DENSE, "B = 65 536: every transform runs as 65 535 + 1 clips", T=8, B=65536,
     n_iter=1)
_row("b65536_128_64", 128, 64, BLK, "B = 65 536 at R = 2 on the block kernel: a deterministic chunked call, compared bit for bit "
     "with its chunks run alone", T=8, B=65536, n_iter=1)


def win_length_of(row):
    return row["win_length"] or row["n_fft"]


def ctor(row):
    """Griffin_Lim constructor arguments of a row."""
    kw = dict(n_fft=row["n_fft"], n_iter=row["n_iter"], hop_length=row["hop"], window=row["window"],
              pad_mode=row["pad_mode"], momentum=row["momentum"])
    if row["win_length"] is not None:
        kw["win_length"] = row["win_length"]
    return kw


def row_block(row):
    """The block-partial layout from the constructor alone: a periodic-Hann DFT the full n_fft wide, at a hop the
    block kernel takes (``dd.row_geometry``'s rule; the module's STFT is never trainable)."""
    return (row["window"] == "hann" and win_length_of(row) == row["n_fft"]
            and bool(_C.block_layout_ok(row["n_fft"], row["hop"])))


def module_block(mod):
    """Whether the module's STFT packs the block-partial layout: its hop fits and its buffers ARE the
    periodic-Hann DFT (``PackedBasis.get``)."""
    from nnaudio_b200.features._common import is_hann_dft

    st = mod._stft
    wcos = st.wcos.detach().reshape(st.wcos.shape[0], -1)
    wsin = st.wsin.detach().reshape(st.wsin.shape[0], -1)
    return bool(_C.block_layout_ok(st.n_fft, st.stride)) and is_hann_dft(wcos, wsin)


def clips_len(row):
    return row["hop"] * (row["T"] - 1)


def problem(row, B=None):
    """(S, phase) float32 (B, n_fft // 2 + 1, T): the magnitude of the STFT of seeded white noise clips of
    hop (T - 1) samples, and a seeded randn initial phase."""
    B = row["B"] if B is None else B
    n_fft, hop = row["n_fft"], row["hop"]
    rng = np.random.RandomState(n_fft * 7 + hop + row["T"] + B % 1000)
    x = rng.standard_normal((B, clips_len(row)))
    win = dd.window(row["window"], n_fft, row["win_length"])
    k = np.arange(n_fft // 2 + 1)[:, None]
    ang = 2.0 * np.pi * ((k * np.arange(n_fft)[None, :]) % n_fft) / n_fft
    S = np.abs(dd.ref_stft(x, np.cos(ang) * win, np.sin(ang) * win, hop, True, row["pad_mode"]))
    assert S.shape[2] == row["T"]
    return S.astype(np.float32), rng.standard_normal(S.shape).astype(np.float32)


# ------------------------------------------------------------------------------------------ launch model ----
def chunks(B):
    return [min(MAX_BATCH, B - i) for i in range(0, B, MAX_BATCH)]


def ola_addends(row):
    """Most fp32 atomic additions onto one overlap-add sample in one inverse: the frames that overlap it times the
    GEMM's K chunks, each of which adds its partial sum on its own."""
    n_fft, hop = row["n_fft"], row["hop"]
    K_gemm = od.istft_operands(1, row["T"], n_fft, n_fft // 2 + 1)[2]
    return min(row["T"], -(-n_fft // hop)) * od.ola_k_splits(K_gemm)


def call_model(row, block=None):
    """What one whole call adds: ``routes`` ({STFT_* route: count}, the forward is n_iter calls per chunk of at
    most 65 535 clips, the inverse moves no STFT route), ``flops`` (the executed MMA flops of n_iter forwards and
    n_iter + 1 inverses, summed over the chunks), the per-call ``fwd_flops`` / ``inv_flops``, the planned forward
    ``route`` and whether two calls are bitwise equal (``deterministic``: the forward's plan says so and no
    overlap-add sample takes more than two atomic additions onto its zero start, since a + b = b + a in IEEE
    arithmetic but (a + b) + c need not equal (a + c) + b).

    ``block``: whether the module packed the block-partial layout (default: ``row_block``)."""
    n_fft, hop, T, n_iter = row["n_fft"], row["hop"], row["T"], row["n_iter"]
    F = n_fft // 2 + 1
    block = row_block(row) if block is None else block
    routes, fwd_flops, inv_flops, planned, det = {}, 0.0, 0.0, set(), True
    for b in chunks(row["B"]):
        p = dd.plan(n_fft, F, hop, b, clips_len(row), True, block)
        assert p["T"] == T
        for r in p["routes"]:
            routes[r] = routes.get(r, 0) + n_iter
            planned.add(r)
        fwd_flops += p["flops"]
        det = det and p["deterministic"]
        inv_flops += od.ola_exec_flops(*od.istft_operands(b, T, n_fft, F))
    assert len(planned) == 1
    routes = {r: n for r, n in routes.items() if n}
    return dict(routes=routes, route=planned.pop(), flops=n_iter * fwd_flops + (n_iter + 1) * inv_flops,
                fwd_flops=fwd_flops, inv_flops=inv_flops, ola_addends=ola_addends(row),
                deterministic=det and ola_addends(row) <= 2)
