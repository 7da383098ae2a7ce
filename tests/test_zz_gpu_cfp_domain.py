"""CFP across its contraction shapes and kernel routes (-m gpu; rows: tests/cfp_domain.py).

Every row runs under path auto and simt with ``_C.cqt1992v2_forward`` wrapped so that each call is recorded and
passed through, and must
- hold each contraction to the float64 contraction of its own fp32 input and banks: ``|y - y64| <= TAU[route] S``
  over the whole output, S the componentwise scale ``|A| . |W_re| + |A| . |W_im|``;
- make exactly the calls of the model, on the routes the model predicts: the CQT1992v2 route counters move by the
  model's sums, the executed-MMA-flop counter by its flop sum, and no STFT or pyramid counter moves;
- match the float64 oracle end to end: tfrL0 (no non-linearity) at 1e-4, Z / tfrLF / tfrLQ at the row's bar,
  outputs that are exactly zero (silence, the ``null`` outputs) exactly;
- give bit-identical results on a second call and for a bf16 / fp16 waveform against its fp32 upcast;
- agree between the two paths on the STFT stage (same input) within the sum of their stage bars."""
import warnings

import numpy as np
import pytest
import torch

import cfp_domain as fd
from conftest import record_error
from helpers import rel_errors
from nnaudio_b200 import _C

pytestmark = pytest.mark.gpu
L0_BAR = 1e-4


def _counts():
    return ([_C.cqt1992v2_route_count(r) for r in range(_C.CQ1992_ROUTES)],
            [_C.stft_route_count(r) for r in range(_C.STFT_ROUTES)],
            [_C.pyramid_route_count(r) for r in range(_C.PYR_ROUTES)])


def _run(mod, x, drop, rec=None, monkeypatch=None):
    """The four outputs of one forward, the CQT1992v2 route deltas, the executed flops and whether any STFT or
    pyramid counter moved; ``rec``: a list each call's (x, w_re, w_im, hop, center, fmt, y) is appended to."""
    real = _C.cqt1992v2_forward

    def recording(x_, k_real, k_imag, packed, k_begin, k_end, hop, center, pad_mode, scale, scale_all, fmt, eps,
                  **kw):
        y = real(x_, k_real, k_imag, packed, k_begin, k_end, hop, center, pad_mode, scale, scale_all, fmt, eps, **kw)
        rec.append((x_, k_real, k_imag, hop, center, fmt, y))
        return y

    if rec is not None:
        monkeypatch.setattr(_C, "cqt1992v2_forward", recording)
    before = _counts()
    _C.profile_read_exec_flops()
    _C.profile_enable(True)
    try:
        with torch.no_grad(), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ys = mod._maps(x, drop)
        torch.cuda.synchronize()
    finally:
        _C.profile_enable(False)
        _C.profile_read()
        if rec is not None:
            monkeypatch.setattr(_C, "cqt1992v2_forward", real)
    flops = _C.profile_read_exec_flops()
    after = _counts()
    routes = {r: a - b for r, (a, b) in enumerate(zip(after[0], before[0])) if a != b}
    return ys, routes, flops, after[1:] != before[1:]


@pytest.mark.parametrize("name", sorted(fd.ROWS))
def test_cfp_domain(name, monkeypatch):
    mod = fd.build_row(name).cuda()
    B, L = fd.ROWS[name][2]
    drop = fd.drops(name)
    opts = fd.row_options(name)
    xn = fd.make_input(name)
    x = torch.from_numpy(xn).cuda()
    want = fd.run_oracle(mod, xn, drop)
    stft_out = {}
    for path in ("auto", "simt"):
        monkeypatch.setenv("NNAUDIO_B200_PATH", path)
        steps = fd.plan(mod, B, L, drop, path)
        want_routes, want_flops = fd.route_totals(steps)
        rec = []
        ys, routes, flops, other = _run(mod, x, drop, rec, monkeypatch)
        case = f"{name}|{path}"
        assert routes == want_routes, (case, routes, want_routes)
        assert flops == want_flops, (case, flops, want_flops)
        assert not other, f"{case}: an STFT or pyramid counter moved"
        assert len(rec) == len(steps), (case, len(rec), len(steps))

        # ---- each contraction against float64
        for i, ((c, r), (xi, wr, wi, hop, center, fmt, y)) in enumerate(zip(steps, rec)):
            assert (tuple(xi.shape), tuple(wr.shape), hop, center, fmt) == \
                ((c["B"], c["L"]), (c["F"], c["K"]), c["hop"], c["center"], c["fmt"]), (case, i, c)
            y64, s = fd.ref_stage(xi, wr, wi, hop, center, fmt)
            assert tuple(y.shape) == tuple(y64.shape), (case, i)
            ratio = fd.stage_ratio(y, y64, s)
            record_error("cfp_domain_stage", f"{case}|{i}|{c['stage']}", route=fd.ROUTE_NAMES[r["route"]],
                         ratio=ratio, tau=fd.TAU[r["route"]])
            assert ratio <= fd.TAU[r["route"]], (case, i, c["stage"], fd.ROUTE_NAMES[r["route"]], ratio)
            del y64, s
        stft_out[path] = (rec[0][6], steps[0][1]["route"])
        first = rec[0][:6]
        del rec

        # ---- end to end against the oracle
        got = [t.cpu().double().numpy() for t in ys]
        for i, (g, w) in enumerate(zip(got, want)):
            assert g.shape == w.shape and np.isfinite(g).all(), (case, i, g.shape, w.shape)
            if not w.size:
                continue
            if i in opts["null"] or not np.abs(w).max():
                if i in opts["null"] and opts["bar"] is None:
                    continue  # exactly zero only in exact arithmetic: the frame mean cancels to round-off
                assert not np.abs(g).max(), (case, i, np.abs(g).max())
                continue
            emax, el2 = rel_errors(g, w)
            record_error("cfp_domain", f"{case}|{i}", max_rel=emax, l2_rel=el2)
            if i == 1:
                assert emax <= L0_BAR and el2 <= L0_BAR, (case, "tfrL0", emax, el2)
            elif opts["bar"] is not None:
                assert emax <= opts["bar"] and el2 <= opts["bar"], (case, i, emax, el2, opts["bar"])

        # ---- repeatable, and 16-bit waveforms read as their fp32 upcast
        again = _run(mod, x, drop)[0]
        assert all(torch.equal(a, b) for a, b in zip(ys, again)), f"{case}: two calls differ"
        if path == "auto":
            for dt in (torch.bfloat16, torch.float16):
                xh = x.to(dt)
                yh = _run(mod, xh, drop)[0]
                y32 = _run(mod, xh.float(), drop)[0]
                assert all(torch.equal(a, b) for a, b in zip(yh, y32)), (case, dt)
        del ys, again
        torch.cuda.empty_cache()

    # ---- the two paths agree on the STFT stage (same input)
    (ya, ra), (ys_, rs) = stft_out["auto"], stft_out["simt"]
    _, s = fd.ref_stage(*first[:3], *first[3:])
    d = (ya.double() - ys_.double()).abs()
    assert float((d / (s + fd.TINY)).max()) <= fd.TAU[ra] + fd.TAU[rs], name
