"""Golden fixtures of ``Combined_Frequency_Periodicity`` / ``CFP`` from the UNMODIFIED reference
(features/cfp.py), run on CPU in the build container.

One environment shim, no source change: the reference calls ``scipy.signal.blackmanharris``
(cfp.py:89), which SciPy >= 1.13 only exposes as ``scipy.signal.windows.blackmanharris`` — the alias is
restored on the ``scipy.signal`` module object before the import.  Everything else (``torch.stft`` with
``return_complex=False``, ``torch.fft.fft`` through ``rfft_fn``) still executes under the image's torch.

  ref_cfp.npz    forward outputs for cases.CFP_CASES
  ref_cfp.json   sha256 of the state_dict buffers, the public attribute surface, constructor / forward
                 signatures, and the exception types of cases.CFP_ERROR_CASES

Run:  PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_cfp.py
"""
from __future__ import annotations

import hashlib
import inspect
import json
import os
import sys
import warnings

import numpy as np
import scipy.signal
import scipy.signal.windows
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ["NNAUDIO_REF"]  # the reference repository's Installation/ directory
sys.dont_write_bytecode = True
sys.path.insert(0, REF)
sys.path.insert(0, HERE)

if not hasattr(scipy.signal, "blackmanharris"):
    scipy.signal.blackmanharris = scipy.signal.windows.blackmanharris  # removed alias, same function

from cases import CFP_CASES, CFP_DESIGN_CASES, CFP_ERROR_CASES, attribute_surface, make_input  # noqa: E402
from nnAudio.features import cfp as ref_cfp  # noqa: E402


def sha(t: torch.Tensor) -> str:
    return hashlib.sha256(np.ascontiguousarray(t.detach().cpu().numpy()).tobytes()).hexdigest()


def main():
    warnings.simplefilter("ignore")
    outputs, meta = {}, {"buffers": {}, "attributes": {}, "signatures": {}, "errors": {}}
    for cid, cls, ctor, inp in CFP_CASES:
        mod = getattr(ref_cfp, cls)(**ctor)
        meta["buffers"][cid] = {k: [list(v.shape), sha(v)] for k, v in mod.state_dict().items()}
        with torch.no_grad():
            y = mod(torch.from_numpy(make_input(inp)))
        meta["attributes"][cid] = attribute_surface(mod)  # after forward: includes `t`
        ys = y if isinstance(y, tuple) else (y,)
        for i, t in enumerate(ys):
            outputs[f"{cid}|{i}"] = t.numpy().astype(np.float32)
            print(f"{cid}|{i}", tuple(t.shape), float(t.abs().max()))
    for cid, cls, ctor in CFP_DESIGN_CASES:
        mod = getattr(ref_cfp, cls)(**ctor)
        meta["buffers"][cid] = {k: [list(v.shape), sha(v)] for k, v in mod.state_dict().items()}
        meta["attributes"][cid] = attribute_surface(mod)
    for cls in ("Combined_Frequency_Periodicity", "CFP"):
        klass = getattr(ref_cfp, cls)
        meta["signatures"][cls] = {
            meth: [[q.name, None if q.default is inspect.Parameter.empty else repr(q.default)]
                   for q in list(inspect.signature(getattr(klass, meth)).parameters.values())[1:]]
            for meth in ("__init__", "forward")}
    for cid, cls, ctor, shape in CFP_ERROR_CASES:
        try:
            mod = getattr(ref_cfp, cls)(**ctor)
            with torch.no_grad():
                mod(torch.zeros(shape))
            meta["errors"][cid] = "ok"
        except Exception as e:  # noqa: BLE001  (the point is to record the type)
            meta["errors"][cid] = type(e).__name__
        print(cid, "->", meta["errors"][cid])
    np.savez_compressed(os.path.join(HERE, "ref_cfp.npz"), **outputs)
    with open(os.path.join(HERE, "ref_cfp.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
