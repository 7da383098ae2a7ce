#!/usr/bin/env python
"""GPU probe: wgmma smem descriptors that start at an arbitrary row of a SWIZZLE_128B block
(nnab_probe_rowoffset, csrc/tc_probe.cu).  Prints, per row offset r, whether
base_offset = 0 and / or base_offset = r & 7 reproduce A[r:r+128] @ B^T.

    python tools/probe_rowoffset.py [result.json]"""
import ctypes, json, os, sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from nnaudio_b200 import _C  # noqa: E402

lib = _C.lib()
lib.nnab_probe_rowoffset.restype = ctypes.c_int
lib.nnab_probe_rowoffset.argtypes = [ctypes.c_void_p] * 4
g = torch.Generator().manual_seed(0)
a = torch.randn(144, 64, generator=g).to(torch.bfloat16).cuda()
b = torch.randn(32, 64, generator=g).to(torch.bfloat16).cuda()
out = torch.zeros(2, 16, 128, 32, device="cuda")
rc = lib.nnab_probe_rowoffset(a.data_ptr(), b.data_ptr(), out.data_ptr(), torch.cuda.current_stream().cuda_stream)
torch.cuda.synchronize()
assert rc == 0, rc
af, bf = a.float().cpu().numpy(), b.float().cpu().numpy()
res = {}
for v in range(2):
    for r in range(16):
        want = af[r:r + 128] @ bf.T
        got = out[v, r].cpu().numpy()
        err = float(np.abs(got - want).max() / np.abs(want).max())
        res[f"v{v}_r{r}"] = err
ok0 = [r for r in range(16) if res[f"v0_r{r}"] < 1e-3]
ok1 = [r for r in range(16) if res[f"v1_r{r}"] < 1e-3]
print("base_offset = 0      correct for r in", ok0)
print("base_offset = r & 7  correct for r in", ok1)
if len(sys.argv) > 1:
    with open(sys.argv[1], "w") as f:
        json.dump({"errors": res, "ok_base0": ok0, "ok_base_r": ok1}, f, indent=1)
