"""CPU checks of tests/dense_domain.py: the float64 reference against the oracle, the choose_bn replica against the
library, the flop model against hand counts, the partial-sum model, and that every row of the matrix builds the
plan it claims (tests/test_zz_gpu_dense_domain.py then holds the GPU to that plan)."""
import numpy as np
import pytest

import dense_domain as dd
from helpers import build, oracle
from nnaudio_b200 import _C


@pytest.mark.parametrize("ctor,center,pad_mode", [
    (dict(n_fft=512, hop_length=160, win_length=400, window="hamming"), True, "reflect"),
    (dict(n_fft=256, hop_length=37, freq_bins=100, freq_scale="log", sr=16000, fmin=60, fmax=7000), True,
     "constant"),
    (dict(n_fft=400, hop_length=100), False, "reflect"),
])
def test_reference_equals_the_oracle(ctor, center, pad_mode):
    mod = build("STFT", dict(ctor, center=center, pad_mode=pad_mode))
    x = np.random.RandomState(3).standard_normal((2, 3001))
    wc, ws = mod.wcos.numpy(), mod.wsin.numpy()
    X = dd.ref_stft(x, wc, ws, ctor["hop_length"], center, pad_mode)
    # float64 bases on both sides: the same sums in another order
    want = oracle.stft(x, ws.astype(np.float64), wc.astype(np.float64), ctor["hop_length"], center, pad_mode,
                       "Complex")
    got = np.stack((X.real, X.imag), -1)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()
    # the oracle in fp32 on the module's buffers
    want32 = oracle.stft(x, ws, wc, ctor["hop_length"], center, pad_mode, "Complex", dtype=np.float32)
    assert np.abs(got - want32).max() <= 1e-6 * np.abs(want).max()


def test_filterbank_and_mfcc_references_equal_the_oracle():
    mod = build("MFCC", dict(sr=16000, n_fft=400, hop_length=160, n_mels=40, n_mfcc=13))
    st, ml = mod.melspec_layer.stft, mod.melspec_layer
    x = np.random.RandomState(5).standard_normal((2, 8000)) * np.array([[1.0], [1e-4]])
    ws, wc, fb = (t.numpy().astype(np.float64) for t in (st.wsin, st.wcos, ml.mel_basis))
    S = dd.ref_filterbank(dd.ref_stft(x, wc, ws, 160), fb, 2.0)
    assert np.allclose(S, oracle.melspectrogram(x, ws, wc, fb, 160), rtol=1e-12, atol=0)
    want = oracle.mfcc(x, ws, wc, fb, 160, 13, 2.0, 1e-10, 1.0, 80.0)
    assert np.abs(dd.ref_mfcc(S, 13, 1e-10, 1.0, 80.0) - want).max() <= 1e-9


def test_fft_reference_equals_the_dense_product():
    win = dd.window("hamming", 1024, 1000)
    n, k = np.arange(1024), np.arange(513)
    ang = 2 * np.pi * ((k[:, None] * n[None, :]) % 1024) / 1024
    x = np.random.RandomState(9).standard_normal((2, 6000))
    a = dd.ref_stft_fft(x, win, 300)
    b = dd.ref_stft(x, np.cos(ang) * win, np.sin(ang) * win, 300)
    assert np.abs(a - b).max() <= 1e-10 * np.abs(b).max()


def test_choose_bn_replica_equals_the_library():
    lib = _C.lib()
    F = np.arange(1, 16386)
    got = np.array([lib.nnab_pack_tile_n(int(f)) for f in F])
    assert (got == np.array([dd.choose_bn(int(f)) for f in F])).all()
    assert lib.nnab_pack_tile_n(1025) == 208 and lib.nnab_pack_tile_n(84) == 176
    fits = np.array([dd.n_tiles(int(f)) <= dd.TC_MAX_N_TILES for f in F])
    # a fitting width exists up to n_fft 32766 (F = 16384); n_fft 32768 needs 129 tiles even at 256
    assert fits[:16384].all() and not fits[16384]


def test_the_unbounded_rule_sent_long_bases_to_the_cuda_core_kernel():
    """The widths the N-tile bound changes: 3512 even n_fft between 16720 and 32734, 20000 and 24576 among them."""
    changed = [n for n in range(2, 32768, 2)
               if -(-(n + 2) // dd.choose_bn_unbounded(n // 2 + 1)) > dd.TC_MAX_N_TILES
               and dd.n_tiles(n // 2 + 1) <= dd.TC_MAX_N_TILES]
    assert len(changed) == 3512 and changed[0] == 16720 and changed[-1] == 32734
    assert {20000, 24000, 24576, 30000, 32000} <= set(changed)
    assert dd.choose_bn_unbounded(12289) == 144 and dd.choose_bn(12289) == 224


def test_flop_model_hand_counts():
    # 512/128 hamming: 1 phase, B*t_slots = 2 * ceil((11597 + 512) / 128) = 190 -> 2 M tiles; 3 tiles of 176; K 512
    p = dd.plan(512, 257, 128, 2, 128 * 90 + 77)
    assert p["flops"] == 6 * 2 * 128 * 3 * 176 * 512
    # 1000/250: 4 phases, hop_eff 1000, t_slots = ceil(23050 / 1000) = 24 -> 48 rows, 1 M tile; 7 x 144; K 1024
    p = dd.plan(1000, 501, 250, 2, 22050)
    assert (p["n_ph"], p["launched"], p["t_slots"]) == (4, 4, 24)
    assert p["flops"] == 4 * 6 * 128 * 7 * 144 * 1024
    # 256/37 center=False, T = 3 < 8 phases: three launches, t_slots = ceil(335 / 296) = 2; 144 x 2; K 256
    p = dd.plan(256, 129, 37, 3, 335, center=False)
    assert (p["T"], p["launched"]) == (3, 3)
    assert p["flops"] == 3 * 6 * 128 * 2 * 144 * 256


def test_partial_sum_counts():
    sums = {name: dd.row_plan(name)["max_sums"] for name in ("mel_3_sums", "mel_4_sums", "mel_16384",
                                                             "mel_fused_speech")}
    assert sums == {"mel_3_sums": 3, "mel_4_sums": 4, "mel_16384": 8, "mel_fused_speech": 2}


@pytest.mark.parametrize("name", sorted(dd.ROWS))
def test_row_builds_the_plan_it_claims(name):
    p = dd.row_plan(name)
    for k, v in dd.ROWS[name][3].items():
        assert p[k] == v, (name, k, p[k], v)
    assert all(n == 1 for n in p["routes"].values())
    fb_routes = {_C.STFT_FB_FUSED, _C.STFT_FB_PLANES, _C.STFT_FB_GEMM}
    assert len(set(p["routes"]) - fb_routes) == 1
    assert len(set(p["routes"]) & fb_routes) == (0 if dd.ROWS[name][0].endswith("STFT") else 1)


def test_the_matrix_reaches_every_route():
    reached = set()
    for name in dd.ROWS:
        reached |= set(dd.row_plan(name)["routes"])
    assert reached == set(range(_C.STFT_ROUTES))
    assert _C.stft_route_count(-1) == 0 and _C.stft_route_count(_C.STFT_ROUTES) == 0
