"""CPU: the argument lists ``_C`` hands to the C ABI for every framed transform in every call mode.

The other host tests replace the ``_C`` wrappers, so the marshalling itself never runs without a GPU.  Here a
recording stand-in takes the place of ``libnnab.so``; the stream, the device context, the workspace and the lane
table copies (which need a device) are replaced, and every pointer argument is mapped back to the name of the
tensor it came from.  Each call must have the arity ``SIGNATURES`` declares, and the transform's arguments between
the waveform head and ``out`` must be the same in the offline, chunk, pool and device-pool calls.
"""
import contextlib
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from nnaudio_b200 import _C

STREAM = 0x5EED


class _Recorder:
    """Stands in for the loaded library: records every call, returns success (and 256 for a size query)."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 256 if name.endswith("_bytes") else 0

        fn.__name__ = name
        return fn


def _tensors():
    g = torch.Generator().manual_seed(0)
    t = lambda *shape: torch.randn(*shape, generator=g)  # noqa: E731
    stft = dict(wcos=t(33, 64), wsin=t(33, 64), packed=t(16), n_fft=64, hop=16, center=True,
                pad_mode=_C.PAD_REFLECT)
    return {
        "stft_forward": dict(stft, out_format=_C.FMT_COMPLEX, sqrt_eps=1e-8),
        "stft_filterbank_forward": dict(stft, sqrt_eps=0.0, power=2.0, fb=t(12, 33), fb_table=t(8)),
        "mfcc_forward": dict(stft, center=False, sqrt_eps=0.0, power=2.0, mel_basis=t(12, 33), amin=1e-10, ref=1.0,
                             top_db=None, dct=t(8, 12), fb_table=None),
        "cqt1992v2_forward": dict(k_real=t(24, 64), k_imag=t(24, 64), packed=t(16),
                                  k_begin=np.arange(24, dtype=np.int32), k_end=np.arange(24, dtype=np.int32) + 40,
                                  hop=16, center=True, pad_mode=_C.PAD_CONSTANT, scale=t(24), scale_all=1.0,
                                  out_format=_C.FMT_MAGNITUDE, sqrt_eps=0.0),
        "cqt_pyramid_forward": dict(banks_real=[t(12, 256), t(12, 128)], banks_imag=[t(12, 256), t(12, 128)],
                                    packed=[t(16), None], lowpass=t(64), lowpass_packed=t(16), early_filter=None,
                                    early_packed=None, early_factor=1, hop=64, pad_mode=_C.PAD_REFLECT, n_bins=24,
                                    scale=t(24), scale_all=1.0, out_format=_C.FMT_COMPLEX, sqrt_eps=0.0),
    }


def _names(**objs):
    """data address -> name of every tensor / numpy array (lists: name[i])."""
    out = {}
    for k, v in objs.items():
        for i, a in enumerate(v if isinstance(v, list) else [v]):
            key = f"{k}[{i}]" if isinstance(v, list) else k
            if isinstance(a, torch.Tensor):
                out[a.data_ptr()] = key
            elif isinstance(a, np.ndarray):
                out[a.ctypes.data] = key
    return out


def _norm(a, names):
    if isinstance(a, ctypes.c_void_p):
        return None if a.value is None else names.get(a.value, "?")
    if isinstance(a, ctypes.Array):
        return [names.get(v, "?") if a._type_ is ctypes.c_void_p and v is not None else v for v in a]
    return a


@contextlib.contextmanager
def _fake_device():
    rec = _Recorder()
    ws = torch.zeros(256, dtype=torch.uint8)
    lanes_dev = []

    def lane_copies(lanes, device):
        if len(lanes) == 0:
            return None, None
        host = torch.as_tensor(lanes, dtype=torch.int64).contiguous()
        lanes_dev.append(host.clone())
        return host, lanes_dev[-1]

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(_C, "lib", lambda: rec)
        mp.setattr(_C, "_stream", lambda device: ctypes.c_void_p(STREAM))
        mp.setattr(_C, "_dev_wave", lambda t, name: t)
        mp.setattr(_C, "_workspace", lambda nbytes, device: (ws, nbytes) if nbytes > 0 else (None, 0))
        mp.setattr(_C, "_lane_copies", lane_copies)
        mp.setattr(torch.cuda, "device", lambda device: contextlib.nullcontext())
        yield rec, ws, lanes_dev


def record():
    """[(mode, C function, arguments with pointers named)] of one call of every transform in every mode."""
    out = []
    x = torch.randn(2, 300, generator=torch.Generator().manual_seed(1))
    ring = torch.zeros(2, 1024)
    lanes = np.array([[0, 100, 40, 3, 300, 0], [1, 50, 20, 1, 120, 1]], np.int64)
    for name, kw in _tensors().items():
        for mode in ("offline", "chunk", "pool", "device"):
            if mode == "device" and name == "cqt_pyramid_forward":
                continue
            with _fake_device() as (rec, ws, lanes_dev):
                operands = {k: v for k, v in kw.items() if isinstance(v, (torch.Tensor, np.ndarray, list))}
                names = _names(x=x, ring=ring, ws=ws, lane_table=lanes, **operands)
                names[STREAM] = "stream"
                if mode == "offline":
                    res = getattr(_C, name)(x, **(dict(kw, T=10) if name == "cqt_pyramid_forward" else kw))
                elif mode == "chunk":
                    st = SimpleNamespace(ring=ring, batch=2, received=100, n_carry=40, frames=3,
                                         dtype=torch.float32)
                    res = getattr(_C, name.replace("_forward", "_chunk_forward"))(st, x, False, 5, **kw)
                elif mode == "pool":
                    pool = SimpleNamespace(ring=ring, slots=2, dtype=torch.float32)
                    res = getattr(_C, name.replace("_forward", "_pool_forward"))(pool, lanes, x, 2, 5, **kw)
                else:
                    fn, res, dws, tail = _C.pool_device_bind(name, kw, 2, 5, torch.device("cpu"))
                    dev = {k: torch.zeros(2, 6, dtype=torch.int64) + i
                           for i, k in enumerate(("counters", "errors", "error_info", "counts", "_lanes"))}
                    pool = SimpleNamespace(ring=ring, slots=2, _fn=fn, _tail=tail, **dev)
                    lengths, end = torch.ones(2, dtype=torch.int32), torch.zeros(2, dtype=torch.bool)
                    assert _C.pool_device_forward(pool, x, lengths, end)
                    names.update(_names(lengths=lengths, end=end, **dev))
                names[res.data_ptr()] = "out"
                names.update({t.data_ptr(): f"lanes_device[{i}]" for i, t in enumerate(lanes_dev)})
                for fn_name, args in rec.calls:
                    out.append((mode, fn_name, [_norm(a, names) for a in args]))
    return out


_HEADS = {"offline": 5, "chunk": 10, "pool": 10, "device": 13}  # waveform head of each mode's forward call


def test_arities_equal_the_signatures_and_every_mode_passes_the_offline_tail():
    calls = record()
    tails = {}
    for mode, name, args in calls:
        assert len(args) == len(_C.SIGNATURES[name][1]), (mode, name, len(args))
        assert "?" not in str(args), (mode, name, args)  # every pointer is one the call was given or made
        if name.endswith("_forward") or name.endswith("_forward_ex"):
            stem = name.replace("nnab_", "").replace("_pool_device_forward", "").replace("_pool_forward", "") \
                .replace("_chunk_forward", "").replace("_forward_ex", "")
            assert args[-1] == "stream" and args[-6] in ("out", None), (mode, name, args)
            tails.setdefault(stem, {})[mode] = args[_HEADS[mode]:-6]
    assert sorted(tails) == ["cqt1992v2", "cqt_pyramid", "mfcc", "stft", "stft_filterbank"]
    for stem, by_mode in tails.items():
        assert set(by_mode) == ({"offline", "chunk", "pool"} | (set() if stem == "cqt_pyramid" else {"device"}))
        for mode, tail in by_mode.items():
            assert tail == by_mode["offline"], (stem, mode, tail, by_mode["offline"])


def test_workspace_queries_take_the_offline_geometry():
    """Every mode asks the workspace size with the transform's (K, F, hop) and the same query tail."""
    calls = [(m, n, a) for m, n, a in record() if n.endswith("_workspace_bytes") and "pyramid" not in n]
    assert len(calls) == 16
    by_stem = {}
    for mode, name, args in calls:
        stem = name.replace("_chunk", "").replace("_pool", "")
        head = {"offline": 2, "chunk": 5, "pool": 2, "device": 2}[mode]
        geometry, rest = args[head:head + 3], args[head + 3:]
        if mode == "offline":
            rest = rest[1:]  # center
        elif mode == "chunk":
            rest = rest[2:]  # center, pad mode
        by_stem.setdefault(stem, set()).add((tuple(geometry), tuple(rest)))
    assert all(len(v) == 1 for v in by_stem.values()), by_stem
