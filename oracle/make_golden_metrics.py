"""Generate tests/golden/metrics.npz by EXECUTING THE REFERENCE'S OWN utils/util.py.

Run in the authoring container only (needs /root/reference with cv2, torchvision and yaml importable):

    python oracle/make_golden_metrics.py

The unmodified utils/util.py is loaded as a module and its ``calculate_psnr`` / ``calculate_ssim`` run on seeded uint8
pairs: uniform noise against a mostly independent mix (low SSIM) and smoothed "natural-ish" fields against a lightly
perturbed copy (high SSIM), at 64x96x3, 37x53x3, 11x11x3 and 9x13x3 (Gaussian SSIM NaN: the [5:-5] crop is empty),
plus a 2-D and an (h, w, 1) pair.  The fixture stores the images, both results per pair, skimage's PSNR expression
(``10*log10(255**2/mse)``, restated: scikit-image is not a dependency) and ``cv2.getGaussianKernel(11, 1.5)``.
Nothing under /root/reference is copied into the repository.
"""
import importlib.util
import os
import warnings

import cv2
import numpy as np
from scipy.ndimage import gaussian_filter

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "metrics.npz")
UTIL = "/root/reference/utils/util.py"


def smooth_field(rng, shape):
    """Band-limited noise stretched to [0, 255]: local structure like a photograph, not white noise."""
    z = gaussian_filter(rng.standard_normal(shape), sigma=(3.0, 3.0) + (0.0,) * (len(shape) - 2))
    z = (z - z.min()) / max(z.max() - z.min(), 1e-9)
    return np.clip(np.round(z * 235 + 10), 0, 255).astype(np.uint8)


def pairs(rng):
    for h, w, c in ((64, 96, 3), (37, 53, 3), (11, 11, 3), (9, 13, 3), (40, 50, 0), (33, 29, 1)):
        shape = (h, w) if c == 0 else (h, w, c)
        a = rng.integers(0, 256, size=shape, dtype=np.uint8)
        u = rng.integers(0, 256, size=shape, dtype=np.uint8)
        b = np.round(0.3 * a + 0.7 * u).astype(np.uint8)                    # mostly independent: SSIM about 0.2-0.3
        yield f"noise_{h}x{w}x{c}", a, b
        if (h, w) in ((64, 96), (37, 53), (40, 50), (33, 29)):
            a = smooth_field(rng, shape)
            b = np.clip(a.astype(np.int32) + rng.normal(0, 3, size=shape).round().astype(np.int32), 0, 255).astype(np.uint8)
            yield f"smooth_{h}x{w}x{c}", a, b


def main():
    spec = importlib.util.spec_from_file_location("reference_util", UTIL)
    util = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(util)
    rng = np.random.default_rng(31)
    rec, names = {}, []
    for name, a, b in pairs(rng):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)        # the empty-slice mean of the 9x13 pair
            s = util.calculate_ssim(a, b)
        p = util.calculate_psnr(a, b)
        mse = np.mean(np.square(a.astype(np.float64) - b.astype(np.float64)), dtype=np.float64)
        rec[f"{name}_a"], rec[f"{name}_b"] = a, b
        rec[f"{name}_psnr"], rec[f"{name}_ssim"] = np.float64(p), np.float64(s)
        rec[f"{name}_psnr_sk"] = np.float64(10 * np.log10((255 ** 2) / mse))
        names.append(name)
        print(f"{name:22s} psnr {p:8.4f}  ssim {s:.6f}")
    rec["names"] = np.array(names)
    rec["gauss11"] = cv2.getGaussianKernel(11, 1.5).ravel()
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
