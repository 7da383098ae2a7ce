"""Host checks of tests/stream_domain.py: every row's chunkings reach the readiness thresholds they claim, a push's
modelled route is the offline call's, the device pools' frame cap is the readiness rule's, the matrix reaches every
stream counter a push can move, and the inverse streams refuse hop > n_fft at construction."""
import warnings

import pytest

import dense_domain as dd
import ola_domain as od
import pyramid_domain as pd
import stream_domain as sd
from helpers import build
from nnaudio_b200 import _C
from nnaudio_b200.streaming import DeviceInversePool, InversePool, StreamingInverse


def _module(name):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return build(sd.base_class(name), sd.constructor(name))


def _cq_width(name):
    return sd.CQ_ROWS[name][4][1] if not sd.is_stft(name) else None


@pytest.mark.parametrize("name", sd.FORWARD)
def test_chunkings_reach_the_thresholds_they_claim(name):
    assert sd.EDGES[name]
    K, hop, pad, reflect = sd.geometry(name, _cq_width(name))
    B, L = sd.clip(name)
    n_ph = dd.num_phases(hop)
    ch = sd.row_chunkings(name, _cq_width(name))
    got = set()
    for sizes in ch.values():
        got |= sd.properties(sizes, K, hop, pad, reflect, n_ph)
    want = {"threshold", "zero_length", "longer_than_K", "two_wraps", "zero_after_frames"}
    if reflect:
        want.add("pad_plus_one")
    if K < sd.LONG_K:
        assert "ragged" in ch
        if pad > 0:
            want.add("shorter_than_K")
        if n_ph > 1:
            want |= {"fewer_than_phases", "more_than_phases"}
    else:  # threshold cuts only: no stream of single samples
        assert set(ch) <= {"threshold", "pad_plus_one"} and all(len(s) < 64 for s in ch.values()), ch.keys()
    if sd.empty_flush_possible(K, hop, pad, reflect, max(L, 2 * K)):
        want.add("empty_flush")
    assert want <= got, (name, want - got)


def test_simulation_is_the_streams_rule():
    """simulate() on a hand count: n_fft 8, hop 2, reflect: frame 0 needs pad + 1 = 5 samples, then one per hop."""
    assert sd.simulate([3, 1, 1, 0, 2, 1], 8, 2, 4, True) == [0, 0, 1, 0, 1, 1, 2]
    assert sd.simulate([3, 1], 8, 2, 0, False) == [0, 0, 0]


@pytest.mark.parametrize("name", [n for n in sd.FORWARD if sd.is_stft(n) and not sd.auto_simt(n)])
def test_stft_push_takes_the_offline_route(name):
    """A push's contraction and filterbank routes are the offline call's, for every push the threshold chunking
    returns frames on (a short push of a multi-phase row launches fewer phases, but the same route)."""
    K, hop, pad, reflect = sd.geometry(name)
    fb = sd.bank(name)
    offline = dd.plan(*_stft_args(name), fb=fb)["routes"]
    for T in set(sd.simulate(sd.row_chunkings(name)["threshold"], K, hop, pad, reflect)) - {0}:
        p = sd.stft_push(name, 2, T, fb)
        assert p["routes"] == offline, (name, T, p["routes"], offline)
        assert p["T"] == T and p["launched"] == min(p["n_ph"], T)


def _stft_args(name):
    K, F, hop, center, _, block, _ = dd.row_geometry(name, sd.STFT_ROWS[name])
    B, L = sd.clip(name)
    return K, F, hop, B, L, center, block, sd.options(name)["path"]


@pytest.mark.parametrize("name", [n for n in sd.FORWARD if not sd.is_direct(n)][::3])
@pytest.mark.parametrize("chunk", [1, 257, 4000])
def test_device_frame_cap_is_the_readiness_rules(name, chunk):
    K, hop, pad, reflect = sd.geometry(name, _cq_width(name))
    pm = _C.PAD_REFLECT if reflect else _C.PAD_CONSTANT
    assert _C.pool_frame_cap(chunk, K, hop, pad, pm) == sd.device_T_cap(chunk, K, hop, pad, reflect), name


def test_the_matrix_reaches_every_stream_counter():
    stft, cq, pyr = set(), set(), set()
    for name in sd.FORWARD:
        if sd.auto_simt(name):
            continue
        K, hop, pad, reflect = sd.geometry(name, _cq_width(name))
        Ts = set(sd.simulate(sd.row_chunkings(name, _cq_width(name))["threshold"], K, hop, pad, reflect)) - {0}
        if sd.is_stft(name):
            fb = sd.bank(name)
            for T in Ts:
                stft |= set(sd.stft_push(name, sd.clip(name)[0], T, fb)["routes"])
        else:
            mod = _module(name)
            ctas = [c for c in sd.options(name)["tall_ctas"] if c] or [None]
            for T in Ts:
                cq.add(sd.cq1992_push(mod, sd.clip(name)[0], T, tall_ctas=ctas[0])["route"])
    for name in sd.PYRAMID:
        if pd.row_options(name)["path"] == "simt":
            continue
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            mod = build(*pd.ROWS[name][:2])
        if not sd.pyramid_streams(mod):
            continue
        F, widths, hop, e, gen = sd.pyramid_geometry(mod)
        pyr |= set(sd.pyramid_push(F, widths, hop, pd.ROWS[name][2], gen == 2, len(widths) - 1 + (e > 1)))
    assert stft == {_C.STFT_BLOCK, _C.STFT_DENSE, _C.STFT_DENSE_SPLITK, _C.STFT_FB_FUSED, _C.STFT_FB_PLANES,
                    _C.STFT_FB_GEMM}, stft
    assert cq == {_C.CQ1992_TALL, _C.CQ1992_TALL_BALANCED, _C.CQ1992_VARN, _C.CQ1992_VARN_SPLITK, _C.CQ1992_DENSE,
                  _C.CQ1992_DENSE_SPLITK}, cq
    assert pyr == {_C.PYR_PLAN_GEN2, _C.PYR_PLAN_GEN1, _C.PYR_OCT_KERNEL, _C.PYR_OCT_DENSE_PLANES,
                   _C.PYR_OCT_DENSE_FP32, _C.PYR_FIR_BANDED, _C.PYR_FIR_DENSE}, pyr


def test_stream_route_count_is_host_only_and_bounded():
    for fam, n in ((_C.ROUTES_STFT, _C.STFT_ROUTES), (_C.ROUTES_CQ1992, _C.CQ1992_ROUTES), (_C.ROUTES_PYR,
                                                                                         _C.PYR_ROUTES)):
        assert _C.stream_route_count(fam, -1) == 0 and _C.stream_route_count(fam, n) == 0
        assert all(_C.stream_route_count(fam, r) >= 0 for r in range(n))
    assert _C.stream_route_count(3, 0) == 0 and _C.stream_route_count(-1, 0) == 0


@pytest.mark.parametrize("name", [n for n in sd.INVERSE if od.ISTFT_ROWS[n]["hop"] > od.ISTFT_ROWS[n]["n_fft"]])
def test_inverse_streams_refuse_hop_over_n_fft(name):
    row = od.ISTFT_ROWS[name]
    from nnaudio_b200 import iSTFT
    m = iSTFT(n_fft=row["n_fft"], hop_length=row["hop"], window=row["window"], center=row["center"], verbose=False)
    for make in (lambda: StreamingInverse(m, 2), lambda: InversePool(m, 2), lambda: DeviceInversePool(m, 2, 4)):
        with pytest.raises(ValueError, match="do not overlap"):
            make()


def test_pyramid_rows_that_stream():
    """The matrix streams gen-2, gen-1 and early-downsampling rows; a row whose octaves frame at different rates is
    refused (by StreamingPyramid, which the GPU test builds)."""
    kinds = set()
    for name in sd.PYRAMID:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            mod = build(*pd.ROWS[name][:2])
        if sd.pyramid_streams(mod):
            _, _, _, e, gen = sd.pyramid_geometry(mod)
            kinds.add((gen, e > 1))
    assert {(2, False), (1, False), (1, True)} <= kinds, kinds
