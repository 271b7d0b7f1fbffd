"""Generate tests/golden/ssim_loss.npz by EXECUTING THE REFERENCE'S OWN utils/util.py.

Run in the authoring container only (needs /root/reference with cv2, torchvision and yaml importable):

    python oracle/make_golden_ssim.py

The unmodified utils/util.py is loaded as a module and its ``ssim`` and ``calculate_ssim`` run on seeded images
scaled by 255 (the reference's data range), 3 channels (h, w, 3): smooth and noisy content, values in [0, 1] and out
to 0.5 beyond, an identical pair and constant pairs (sigma = 0), at 11x11, 12x13, 24x31 and 37x53.  The images hold
fp32 values (so an fp32 loss sees exactly what the reference saw); the fixture stores them in [0, 1] scale,
(3, h, w), with both results per pair, and ``oracle/ssim_oracle.py`` is pinned to them at data range 1.  Nothing
under /root/reference is copied into the repository.
"""
import importlib.util
import os

import numpy as np
from scipy.ndimage import gaussian_filter

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "ssim_loss.npz")
UTIL = "/root/reference/utils/util.py"


def smooth(rng, h, w):
    z = gaussian_filter(rng.standard_normal((3, h, w)), sigma=(0, 2.5, 2.5))
    return (z - z.min()) / max(z.max() - z.min(), 1e-9)


def pairs(rng):
    for h, w in ((11, 11), (12, 13), (24, 31)):
        a = rng.random((3, h, w))
        yield f"noise_{h}x{w}", a, 0.4 * a + 0.6 * rng.random((3, h, w))
        a = smooth(rng, h, w)
        yield f"smooth_{h}x{w}", a, np.clip(a + rng.normal(0, 0.02, a.shape), 0, 1)
        a = smooth(rng, h, w) * 2.0 - 0.5                                   # [-0.5, 1.5]
        yield f"wide_{h}x{w}", a, a + rng.normal(0, 0.1, a.shape)
    a = smooth(rng, 37, 53)
    yield "smooth_37x53", a, np.clip(a + rng.normal(0, 0.05, a.shape), 0, 1)
    a = smooth(rng, 24, 31)
    yield "identical_24x31", a, a.copy()
    yield "constant_24x31", np.full((3, 24, 31), 0.25), np.full((3, 24, 31), 0.75)
    yield "constant_vs_smooth_24x31", np.full((3, 24, 31), 0.5), smooth(rng, 24, 31)


def main():
    spec = importlib.util.spec_from_file_location("reference_util", UTIL)
    util = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(util)
    rng = np.random.default_rng(47)
    rec, names = {}, []
    for name, a, b in pairs(rng):
        a, b = a.astype(np.float32).astype(np.float64), b.astype(np.float32).astype(np.float64)   # fp32-exact values
        x, y = np.ascontiguousarray(a.transpose(1, 2, 0) * 255), np.ascontiguousarray(b.transpose(1, 2, 0) * 255)
        rec[f"{name}_a"], rec[f"{name}_b"] = a.astype(np.float32), b.astype(np.float32)
        rec[f"{name}_ssim"] = np.float64(util.ssim(x, y))
        rec[f"{name}_calc"] = np.float64(util.calculate_ssim(x, y))
        names.append(name)
        print(f"{name:26s} ssim {rec[f'{name}_ssim']:.15f}")
    rec["names"] = np.array(names)
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
