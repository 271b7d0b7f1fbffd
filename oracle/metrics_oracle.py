"""fp64 numpy restatements of the evaluation-loop metrics -- TEST INFRASTRUCTURE ONLY.

* ``psnr`` / ``ssim_gauss11``: utils/util.py:201-231 (``calculate_psnr`` / ``ssim``).  Pinned against the reference's
  own code: ``oracle/make_golden_metrics.py`` runs the unmodified utils/util.py on seeded pairs and stores the results
  in ``tests/golden/metrics.npz``.  The reference filters with ``cv2.filter2D`` and the 2-D outer-product window; this
  restatement uses the separable form (the window is an outer product, and the cropped region never sees a border).
* ``psnr_skimage`` / ``ssim_box7``: ``skimage.measure.compare_psnr`` / ``compare_ssim`` (scikit-image <= 0.17) with
  the defaults test.py:33-35 uses.  scikit-image removed both functions in 0.18 and is not a dependency here, so these
  are restated from skimage's documented algorithm (7x7 uniform window, sample covariance 49/48, K1 = 0.01,
  K2 = 0.03, data range 255 for uint8, map cropped by 3, per-channel means averaged) and pinned analytically rather
  than against skimage itself: identical images give 1, constant images a, b give (2ab+C1)/(a^2+b^2+C1).

Every function takes uint8 numpy arrays (h, w) or (h, w, c) and works in float64 like the code it restates.
"""
from __future__ import annotations

import math

import numpy as np
from scipy.ndimage import correlate1d, uniform_filter

# cv2.getGaussianKernel(11, 1.5) bit for bit (stored in tests/golden/metrics.npz as well)
GAUSS11 = np.array([float.fromhex(h) for h in (
    "0x1.0d956b52a1d6ep-10", "0x1.f1fe01ae5a5b5p-8", "0x1.26eb175d83f66p-5", "0x1.bff0fe8e98418p-4",
    "0x1.b43c3f52b19f3p-3", "0x1.106560aa892bfp-2", "0x1.b43c3f52b19f3p-3", "0x1.bff0fe8e98418p-4",
    "0x1.26eb175d83f66p-5", "0x1.f1fe01ae5a5b5p-8", "0x1.0d956b52a1d6ep-10")])
C1 = (0.01 * 255) ** 2
C2 = (0.03 * 255) ** 2


def _channels(x: np.ndarray):
    x = np.asarray(x)
    return [x] if x.ndim == 2 else [x[:, :, k] for k in range(x.shape[2])]


def psnr(a, b) -> float:
    """utils/util.py:201-208"""
    mse = np.mean((np.asarray(a).astype(np.float64) - np.asarray(b).astype(np.float64)) ** 2)
    if mse == 0:
        return float("inf")
    return 20 * math.log10(255.0 / math.sqrt(mse))


def psnr_skimage(a, b) -> float:
    """skimage <= 0.17 compare_psnr(im_true, im_test) for uint8: 10 log10(data_range^2 / mse), data_range = 255."""
    err = np.mean(np.square(np.asarray(a).astype(np.float64) - np.asarray(b).astype(np.float64)), dtype=np.float64)
    return float("inf") if err == 0 else float(10 * np.log10((255 ** 2) / err))


def ssim_gauss11(a, b) -> float:
    """utils/util.py:211-231 over all channels (cv2.filter2D filters each channel); NaN if h or w < 11."""
    maps = []
    for x, y in zip(_channels(a), _channels(b)):
        x, y = x.astype(np.float64), y.astype(np.float64)

        def filt(z):
            return correlate1d(correlate1d(z, GAUSS11, axis=0), GAUSS11, axis=1)[5:-5, 5:-5]
        mu1, mu2 = filt(x), filt(y)
        mu1_sq, mu2_sq, mu1_mu2 = mu1 ** 2, mu2 ** 2, mu1 * mu2
        sigma1_sq = filt(x ** 2) - mu1_sq
        sigma2_sq = filt(y ** 2) - mu2_sq
        sigma12 = filt(x * y) - mu1_mu2
        maps.append(((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2)))
    m = np.stack(maps)
    return float("nan") if m.size == 0 else float(m.mean())


def ssim_box7(a, b) -> float:
    """skimage <= 0.17 compare_ssim(X, Y) for 2-D uint8 input, or compare_ssim(X, Y, multichannel=True) for (h, w, c)."""
    vals = []
    for x, y in zip(_channels(a), _channels(b)):
        x, y = x.astype(np.float64), y.astype(np.float64)
        cov_norm = 49 / 48                                        # use_sample_covariance=True
        ux, uy = uniform_filter(x, size=7), uniform_filter(y, size=7)
        uxx, uyy, uxy = uniform_filter(x * x, size=7), uniform_filter(y * y, size=7), uniform_filter(x * y, size=7)
        vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
        A1, A2, B1, B2 = 2 * ux * uy + C1, 2 * vxy + C2, ux ** 2 + uy ** 2 + C1, vx + vy + C2
        S = (A1 * A2) / (B1 * B2)
        vals.append(S[3:-3, 3:-3].mean())
    return float(np.mean(vals))
