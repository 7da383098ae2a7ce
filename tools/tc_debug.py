"""GPU debugging aid: run one module on both kernel families and print where
(which bins / frames / clips) the tensor-core path deviates from the SIMT path."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nnaudio_b200 as nb  # noqa: E402


def run(mod, x, path, **kw):
    os.environ["NNAUDIO_B200_PATH"] = path
    with torch.no_grad():
        y = mod(x, **kw)
    torch.cuda.synchronize()
    return y.float().cpu().numpy()


def report(name, a, b):
    d = np.abs(a.astype(np.float64) - b)
    scale = np.abs(b).max()
    print(f"{name}: shape {a.shape} max-rel {d.max() / scale:.3e} l2-rel "
          f"{np.linalg.norm(d) / np.linalg.norm(b):.3e} nan={np.isnan(a).sum()}")
    if d.max() / scale > 1e-4:
        e = d.reshape(d.shape[0], d.shape[1], d.shape[2], -1).max(-1) / scale
        print("  per-clip max:", np.round(e.max((1, 2)), 5))
        fb = e.max((0, 2))
        print("  per-bin-block(16) max:", np.round([fb[i:i + 16].max() for i in range(0, len(fb), 16)], 4))
        tb = e.max((0, 1))
        print("  per-frame-block(16) max:", np.round([tb[i:i + 16].max() for i in range(0, len(tb), 16)], 4))


def main():
    torch.manual_seed(0)
    cases = [
        ("stft512/256", nb.STFT(n_fft=512, hop_length=256, verbose=False), (2, 16000), dict(output_format="Complex")),
        ("stft2048/512", nb.STFT(n_fft=2048, hop_length=512, verbose=False), (3, 44100), dict(output_format="Complex")),
        ("stft1024/160 (overlap map)", nb.STFT(n_fft=1024, hop_length=160, verbose=False), (2, 16000), dict(output_format="Magnitude")),
        ("mel cfg2 x4", nb.MelSpectrogram(sr=22050, n_fft=2048, hop_length=512, n_mels=128, verbose=False), (4, 220500), {}),
        ("cqt1992v2 84", nb.CQT1992v2(sr=44100, n_bins=84, fmin=32.7, verbose=False), (2, 100000), dict(output_format="Complex")),
        ("stft512/100 (2 phases)", nb.STFT(n_fft=512, hop_length=100, verbose=False), (2, 16000), dict(output_format="Complex")),
        ("stft256/37 (8 phases)", nb.STFT(n_fft=256, hop_length=37, verbose=False), (2, 9000), dict(output_format="Magnitude")),
        ("cqt2010v2 pyramid", nb.CQT2010v2(sr=22050, n_bins=88, verbose=False), (3, 65536), dict(output_format="Complex")),
        ("vqt pyramid", nb.VQT(sr=22050, gamma=3, verbose=False), (2, 65536), dict(output_format="Magnitude")),
    ]
    only = [a for a in sys.argv[1:] if not a.startswith('--')] or None
    for name, mod, shape, kw in cases:
        if only and not any(o in name for o in only):
            continue
        mod = mod.cuda()
        x = torch.randn(*shape, device="cuda")
        ref = run(mod, x, "simt", **kw)
        try:
            got = run(mod, x, "tc", **kw)
        except Exception as e:  # noqa: BLE001
            print(f"{name}: tensor-core path raised {type(e).__name__}: {e}")
            continue
        report(name, got, ref)
        if "--oracle" in sys.argv:
            sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
            from helpers import run_oracle
            orc = run_oracle(type(mod).__name__, mod, x.cpu().numpy(), kw)
            report(name + " [tensor-core vs fp64 oracle]", got, orc)
            report(name + " [simt    vs fp64 oracle]", ref, orc)


if __name__ == "__main__":
    main()
