"""GPU parity of Combined_Frequency_Periodicity / CFP (-m gpu; collected last): the three contraction
stages run on the tensor-core framed kernel (and, as the cross-check, on the fp32 CUDA-core kernel) through
the C ABI, against the unmodified reference's outputs (tests/golden/ref_cfp.npz) and the CPU oracle.

Tolerances.  CFP raises magnitudes to small powers (|X|^0.24, ceps^0.6) and, with a zero exponent, takes
log(relu(.) + 1e-8): errors of the contractions (~5e-6 of the largest term for the split-bf16 tensor path,
the same order for an fp32 dot product of 4000 terms) are amplified near zero.  tools/sim_cfp_split.py
predicts the tensor path's error per case on the CPU (bf16 hi/lo emulation through OUR host layer):
<= 2.8e-5 for the default three-layer configurations, 7.4e-5 with four layers, 1.1e-4 with a log layer.
The default configurations are held to the 1e-4 bar of the other modules; the two deliberately
ill-conditioned ones to 3e-4 / 5e-4 (about 4x the prediction)."""
import os
import warnings

import numpy as np
import pytest
import torch

from conftest import record_error
from helpers import GOLDEN, build, oracle, rel_errors
from cases import CFP_CASES, make_input

pytestmark = pytest.mark.gpu
TOL = {"cfp_fr4_four_layers": 3e-4, "cfp_odd_n_log_layer": 5e-4}


def _run(mod, x, path):
    os.environ["NNAUDIO_B200_PATH"] = path
    try:
        with torch.no_grad(), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            y = mod(torch.from_numpy(np.ascontiguousarray(x)).cuda())
        torch.cuda.synchronize()
    finally:
        os.environ.pop("NNAUDIO_B200_PATH", None)
    ys = y if isinstance(y, tuple) else (y,)
    return [t.cpu().numpy() for t in ys]


@pytest.mark.parametrize("path", ["auto", "simt"])
@pytest.mark.parametrize("case", CFP_CASES, ids=[c[0] for c in CFP_CASES])
def test_cfp_matches_reference_and_oracle(case, path):
    cid, cls, ctor, inp = case
    mod = build(cls, ctor).cuda()
    x = make_input(inp)
    got = _run(mod, x, path)
    ref = dict(np.load(os.path.join(GOLDEN, "ref_cfp.npz")))
    drop = cls == "Combined_Frequency_Periodicity"
    orc = oracle.cfp(x, mod.h.cpu().numpy(), mod.freq2logfreq_matrix.cpu().numpy(),
                     mod.quef2logfreq_matrix.cpu().numpy(), mod.N, mod.hop_length, mod.g, mod.tc_idx,
                     mod.fc_idx, mod.HighFreqIdx, mod.HighQuefIdx, drop_edge_frames=drop)
    tol = TOL.get(cid, 1e-4)
    assert len(got) == (4 if drop else 1)
    for i, y in enumerate(got):
        want = ref[f"{cid}|{i}"]
        assert y.shape == want.shape, "frame / band indexing must match the reference exactly"
        assert np.isfinite(y).all()
        for name, r in (("reference", want), ("oracle", orc[i])):
            emax, el2 = rel_errors(y, r)
            record_error("cfp", f"{cid}|{i}|{path}|{name}", max_rel=emax, l2_rel=el2, tol=tol)
            assert emax < tol and el2 < tol, (cid, i, path, name, emax, el2)


def test_cfp_runs_on_the_library_and_is_repeatable():
    """The contractions go through libnnab.so (launch counter) and two runs are bit-identical."""
    from nnaudio_b200 import _C

    mod = build("CFP", {}).cuda()
    x = torch.from_numpy(make_input(("randn", 45, (2, 8000)))).cuda()
    before = _C.launch_count()
    with torch.no_grad():
        a = mod(x)
        b = mod(x)
    torch.cuda.synchronize()
    assert _C.launch_count() - before >= 2 * 5  # STFT + two cosine stages + two map products per call
    assert torch.equal(a, b)
