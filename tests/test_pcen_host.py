"""No-GPU checks of PCEN (nnaudio_b200.pcen): the smoothing coefficient, the constructor's refusals, the
state_dict layout, the refusals of CPU tensors and of frames that require grad, the host-side argument checks of
the C entry points, and the float64 reference itself against a direct loop and scipy's lfilter."""
import ctypes
import math

import numpy as np
import pytest
import torch

import pcen_domain as pd
from nnaudio_b200 import _C
from nnaudio_b200.pcen import PCEN, PCENStream, smoothing_coef

EINVAL, OK = -1, 0


def test_smoothing_coef_formula():
    for sr, hop, tc in ((22050, 512, 0.4), (16000, 160, 0.4), (16000, 128, 0.06), (8000, 1, 2.0)):
        t = tc * sr / hop
        s = smoothing_coef(sr, hop, tc)
        assert s == pytest.approx((math.sqrt(1 + 4 * t * t) - 1) / (2 * t * t), rel=1e-15)
        assert t * t * s * s + s - 1 == pytest.approx(0.0, abs=1e-12)  # the root of t^2 s^2 + s = 1 in (0, 1]
        assert 0 < s <= 1
    assert float(PCEN().s) == pytest.approx(smoothing_coef(22050, 512, 0.4), rel=1e-7)
    assert float(PCEN(sr=16000, hop_length=160).s) == pytest.approx(smoothing_coef(16000, 160, 0.4), rel=1e-7)
    assert float(PCEN(s=0.25).s) == 0.25
    with pytest.raises(ValueError):
        smoothing_coef(16000, 0, 0.4)
    with pytest.raises(ValueError):
        smoothing_coef(16000, 160, 0.0)


def test_defaults_follow_librosa():
    m = PCEN()
    assert (float(m.gain), float(m.bias), float(m.power), m.eps) == pytest.approx((0.98, 2.0, 0.5, 1e-6))
    assert all(getattr(m, n).shape == () for n in pd.PARAMS)
    mc = PCEN(n_channels=40, gain=np.linspace(0.5, 1.0, 40))
    assert all(getattr(mc, n).shape == (40,) for n in pd.PARAMS)
    assert torch.allclose(mc.gain, torch.linspace(0.5, 1.0, 40))
    assert torch.all(mc.bias == 2.0)


@pytest.mark.parametrize("kw", [dict(s=0.0), dict(s=1.5), dict(s=-0.1), dict(gain=-0.01), dict(bias=0.0),
                                dict(bias=-1.0), dict(power=0.0), dict(eps=0.0), dict(eps=-1e-6),
                                dict(gain=float("nan")), dict(n_channels=0), dict(time_constant=0.0),
                                dict(n_channels=4, bias=[1.0, 2.0, 0.0, 1.0]), dict(n_channels=4, gain=[1.0, 2.0]),
                                dict(gain=[0.5, 0.6])])
def test_constructor_refusals(kw):
    with pytest.raises(ValueError):
        PCEN(**kw)


def test_constructor_accepts_the_boundaries():
    PCEN(s=1.0, gain=0.0)
    PCEN(n_channels=3, s=[0.1, 0.5, 1.0], power=[0.1, 1.0, 2.0])


@pytest.mark.parametrize("n_channels", [None, 8])
def test_state_dict_keys(n_channels):
    frozen = PCEN(n_channels=n_channels)
    trained = PCEN(n_channels=n_channels, trainable=True)
    assert sorted(frozen.state_dict()) == sorted(trained.state_dict()) == sorted(pd.PARAMS)
    assert dict(frozen.named_parameters()) == {}
    assert sorted(n for n, _ in trained.named_parameters()) == sorted(pd.PARAMS)
    assert all(p.requires_grad for p in trained.parameters())
    assert sorted(n for n, _ in frozen.named_buffers()) == sorted(pd.PARAMS)
    # the keys load across the two kinds
    trained.load_state_dict(frozen.state_dict())


def test_cpu_tensors_have_no_fallback():
    m = PCEN()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m(torch.ones(1, 4, 10))
    with pytest.raises(TypeError):
        m(np.ones((1, 4, 10), np.float32))
    st = PCENStream(m, 2)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        st.step(torch.ones(1, 4, 10))


def test_stream_refuses_grad():
    st = PCENStream(PCEN(), 2)
    with pytest.raises(NotImplementedError, match="forward-only"):
        st.step(torch.ones(1, 4, 10, requires_grad=True))
    with pytest.raises(TypeError):
        PCENStream(torch.nn.Identity(), 2)
    with pytest.raises(ValueError):
        PCENStream(PCEN(), 0)


def _fwd(lib, E=256, B=2, C=4, T=10, prm=512, stride=1, eps=1e-6, P=768, M=None, state=None, primed=None,
         slots=0, row_slot=None, counts=None):
    p = lambda v: None if v is None else ctypes.c_void_p(v)  # noqa: E731  (never dereferenced on the host)
    return lib.nnab_pcen_forward(p(E), B, C, T, p(prm), p(prm), p(prm), p(prm), stride, eps, p(P), p(M), p(state),
                                 p(primed), slots, p(row_slot), p(counts), None)


def test_entry_points_check_arguments_on_the_host():
    lib = _C.lib()
    assert lib.nnab_abi_version() == 1
    assert _fwd(lib, E=None) == EINVAL
    assert _fwd(lib, P=None) == EINVAL
    assert _fwd(lib, prm=None) == EINVAL
    assert _fwd(lib, stride=2) == EINVAL, "the parameter stride is 0 (scalars) or 1 (per channel)"
    assert _fwd(lib, eps=0.0) == EINVAL
    assert _fwd(lib, eps=float("inf")) == EINVAL
    assert _fwd(lib, B=-1) == EINVAL
    assert _fwd(lib, C=0) == EINVAL
    assert _fwd(lib, T=-1) == EINVAL
    assert _fwd(lib, state=1024, slots=4) == EINVAL, "state without primed flags"
    assert _fwd(lib, counts=1024) == EINVAL, "counts belong to a streamed call"
    assert _fwd(lib, row_slot=1024) == EINVAL, "a row map belongs to a streamed call"
    assert _fwd(lib, state=1024, primed=2048, slots=0) == EINVAL
    assert _fwd(lib, B=5, state=1024, primed=2048, slots=4) == EINVAL, "more rows than slots without a row map"
    assert _fwd(lib, M=4096, state=1024, primed=2048, slots=4) == EINVAL, "M belongs to the training call"
    x = ctypes.c_void_p(256)
    bwd = lambda E=x, M=x, g=x, C=4, stride=0, eps=1e-6: lib.nnab_pcen_backward(  # noqa: E731
        E, M, g, 2, C, 10, x, x, x, x, stride, eps, x, x, x, 1 << 20, None)
    assert bwd(E=None) == EINVAL and bwd(M=None) == EINVAL and bwd(g=None) == EINVAL
    assert bwd(C=0) == EINVAL and bwd(stride=-1) == EINVAL and bwd(eps=-1.0) == EINVAL
    assert lib.nnab_pcen_reset(None, None, 4, 8, None) == EINVAL
    assert lib.nnab_pcen_reset(x, None, 0, 8, None) == EINVAL
    assert lib.nnab_pcen_reset(x, None, 4, 0, None) == EINVAL
    assert lib.nnab_pcen_workspace_bytes(3, 40) == 4 * 3 * 40 * 4
    if not torch.cuda.is_available():
        for rc in (_fwd(lib), _fwd(lib, state=1024, primed=2048, slots=4, counts=4096), bwd(),
                   lib.nnab_pcen_reset(x, None, 4, 8, None)):
            assert rc in (-3, -4), rc  # NNAB_EARCH / NNAB_ECUDA: never NNAB_OK without a device
            assert lib.nnab_strerror(rc) != b"ok"


@pytest.mark.parametrize("kind", ["scalar", "channel"])
def test_reference_smoother_matches_loop_and_lfilter(kind):
    E = pd.spectrogram(3, 5, 97, seed=1, lo=-3, hi=3).astype(np.float64)
    s = pd.parameters(kind, 5)[0]
    loop, filt = pd.smoother_loop(E, s), pd.smoother(E, s)
    assert np.allclose(loop, filt, rtol=1e-12, atol=0)
    # the first frame starts settled: M[0] = E[0]
    assert np.allclose(filt[:, :, 0], E[:, :, 0], rtol=1e-14, atol=0)
    # a constant input stays put
    const = np.full((1, 5, 50), 3.5)
    assert np.allclose(pd.smoother(const, s), 3.5, rtol=1e-14, atol=0)


@pytest.mark.parametrize("kind", ["scalar", "channel"])
def test_reference_forms_agree(kind):
    """The expm1 / log1p form of the reference equals the difference form in float64, and the differentiable
    torch reference equals the NumPy one."""
    C = 6
    E = pd.spectrogram(2, C, 40, seed=2, lo=-4, hi=4).astype(np.float64)
    prm = pd.parameters(kind, C)
    P, M, u = pd.reference(E, *prm, 1e-6)
    col = lambda v: pd._per_channel(v, C)[None, :, None]  # noqa: E731
    direct = (col(prm[2]) + u) ** col(prm[3]) - col(prm[2]) ** col(prm[3])
    assert np.allclose(P, direct, rtol=1e-9, atol=1e-12 * np.abs(P).max())
    t = lambda v: torch.tensor(v, dtype=torch.float64)  # noqa: E731
    Pt = pd.reference_torch(t(E), *(t(v) for v in prm), 1e-6)
    assert np.allclose(Pt.numpy(), P, rtol=1e-12, atol=0)


def test_naive_form_cancels_in_fp32():
    """Where u << bias the float32 difference form loses digits the expm1 / log1p form keeps (the GPU test holds
    the kernel to 1e-5 on these entries)."""
    E = np.full((1, 1, 8), 1e-9)
    P, M, u = pd.reference(E, 0.05, 0.98, 2.0, 0.5, 1e-6)
    assert (u / 2.0 < 1e-3).all()
    naive = pd.naive_fp32(torch.tensor(E, dtype=torch.float32), torch.tensor(M, dtype=torch.float32), 0.98, 2.0,
                          0.5, 1e-6).double().numpy()
    assert np.abs(naive - P).max() / np.abs(P).max() > 1e-4
