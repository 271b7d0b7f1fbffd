"""Evaluation metrics of the caller loop on the GPU: test.py:404-458 scores every window with PSNR and SSIM.

``image_metrics`` runs one sm_90a kernel pair (bin_image_metrics_u8) over a uint8 pair and returns its mean |a-b|,
MSE, Gaussian-11 SSIM (utils/util.py:211-231) and box-7 SSIM (skimage <= 0.17 compare_ssim defaults).  PSNR is
computed on the host from the exact integer sum of squares with the reference's own expressions, so it equals the
reference bit for bit.  ``image_metrics_batch`` scores up to 16 pairs per launch and leaves the sums on the device, so
an evaluation loop reads them one window late instead of synchronising per call.

Drop-ins with the reference's names, signatures and return conventions:
  * ``calculate_psnr`` / ``calculate_ssim``  -- utils/util.py:201-250 (test.py:39-40, use_default_ssim = 0);
  * ``compare_psnr`` / ``compare_ssim``      -- skimage.measure of scikit-image <= 0.17 (test.py:33-35), which
    scikit-image 0.18 removed.  ``install_skimage_measure()`` makes test.py's import resolve to them.
Only uint8 images and the default options test.py uses are supported; anything else raises BinB200Error.  CUDA only:
there is no CPU path."""
from __future__ import annotations

import ctypes as C
import math
import sys
import types

import numpy as np
import torch

from ._lib import BIN_METRICS_BGR, BIN_METRICS_MAX_BATCH, BinB200Error, check, lib

_DIMS_MSG = "Input images must have the same dimensions."      # utils/util.py:240, skimage _assert_compatible


def _to_cuda_u8(x, fn: str) -> torch.Tensor:
    if isinstance(x, torch.Tensor):
        if x.dtype != torch.uint8:
            raise BinB200Error(f"{fn}: uint8 images only, got {x.dtype}")
        if not x.is_cuda:
            raise BinB200Error(f"{fn}: CPU tensor given; pass a CUDA tensor or a numpy array (bin_b200 has no CPU path)")
        return x.contiguous()
    x = np.asarray(x)
    if x.dtype != np.uint8:
        raise BinB200Error(f"{fn}: uint8 images only, got {x.dtype}")
    if not torch.cuda.is_available():
        raise BinB200Error(f"{fn}: no CUDA device (bin_b200 has no CPU path)")
    return torch.from_numpy(np.ascontiguousarray(x)).to(torch.cuda.current_device())


def _metric_sums(a, b, fn: str):
    """-> (sum |a-b| as int, sum (a-b)^2 as int, Gaussian SSIM, box SSIM, element count)."""
    if tuple(a.shape) != tuple(b.shape):
        raise ValueError(_DIMS_MSG)
    shape = tuple(a.shape)
    if len(shape) == 2:
        c = 1
    elif len(shape) == 3 and shape[2] in (1, 3):
        c = shape[2]
    else:
        raise BinB200Error(f"{fn}: images must be (h, w), (h, w, 1) or (h, w, 3), got {shape}")
    ta, tb = _to_cuda_u8(a, fn), _to_cuda_u8(b, fn)
    if ta.device != tb.device:
        raise BinB200Error(f"{fn}: images on different devices ({ta.device}, {tb.device})")
    from .rdn import _workspace
    h, w = shape[0], shape[1]
    L = lib()
    with torch.cuda.device(ta.device):
        ws = _workspace(ta.device, max(int(L.bin_image_metrics_workspace_bytes(h, w)), 1))
        out = torch.empty(4, dtype=torch.float64, device=ta.device)
        check(L.bin_image_metrics_u8(ta.data_ptr(), tb.data_ptr(), h, w, c, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                     torch.cuda.current_stream().cuda_stream))
        s_abs, s_sq, g, bx = out.tolist()
    return int(s_abs), int(s_sq), g, bx, h * w * c


def image_metrics(a, b):
    """a, b: uint8 CUDA tensors or numpy arrays, (h, w) or (h, w, c) with c = 1 or 3, h, w >= 7 (numpy inputs are
    uploaded to the current device).  Runs on the current stream.  -> (mean |a-b|, MSE, Gaussian-11 SSIM (NaN if h or
    w < 11), box-7 SSIM), all Python floats."""
    s_abs, s_sq, g, bx, n = _metric_sums(a, b, "image_metrics")
    return s_abs / n, s_sq / n, g, bx


def image_metrics_batch(pairs, bgr: bool = False) -> torch.Tensor:
    """pairs: (a, b) uint8 CUDA tensors, all (h, w) or all (h, w, c) of one shape on one device, c = 1 or 3, h, w >= 7;
    pairs may share a tensor.  Enqueues bin_image_metrics_batch_u8 on the current stream, one tile and one reduce launch
    per BIN_METRICS_MAX_BATCH pairs, and returns at once, with no host synchronisation: a float64 (n, 4) device tensor
    whose row i is { sum |a-b|, sum (a-b)^2, Gaussian-11 SSIM, box-7 SSIM } of pair i, the bits image_metrics' sums
    come from.  bgr=True (c = 3) scores each image as its channel-reversed view: a BGR image (cv2, tensor2img_u8) gets
    exactly the values of its RGB array, which is what test.py scores (read_image_np, test.py:58-66)."""
    pairs = [tuple(p) for p in pairs]
    if not pairs or any(len(p) != 2 for p in pairs):
        raise BinB200Error("image_metrics_batch: give one or more (a, b) pairs")
    first = pairs[0][0]
    for x in (t for p in pairs for t in p):
        if not isinstance(x, torch.Tensor) or not x.is_cuda or x.dtype != torch.uint8:
            raise BinB200Error("image_metrics_batch: uint8 CUDA tensors only")
        if x.shape != first.shape:
            raise ValueError(_DIMS_MSG)
        if x.device != first.device:
            raise BinB200Error(f"image_metrics_batch: images on different devices ({first.device}, {x.device})")
    shape = tuple(first.shape)
    if len(shape) == 2:
        c = 1
    elif len(shape) == 3 and shape[2] in (1, 3):
        c = shape[2]
    else:
        raise BinB200Error(f"image_metrics_batch: images must be (h, w), (h, w, 1) or (h, w, 3), got {shape}")
    if bgr and c != 3:
        raise BinB200Error("image_metrics_batch: bgr=True needs (h, w, 3) images")
    h, w = shape[0], shape[1]
    L = lib()
    flags = BIN_METRICS_BGR if bgr else 0
    with torch.cuda.device(first.device):
        imgs = [(a.contiguous(), b.contiguous()) for a, b in pairs]
        out = torch.empty((len(pairs), 4), dtype=torch.float64, device=first.device)
        stream = torch.cuda.current_stream()
        for k in range(0, len(imgs), BIN_METRICS_MAX_BATCH):
            group = imgs[k:k + BIN_METRICS_MAX_BATCH]
            n = len(group)
            ws = torch.empty(max(int(L.bin_image_metrics_batch_workspace_bytes(n, h, w)), 8), dtype=torch.uint8,
                             device=first.device)
            pa = (C.c_void_p * n)(*[a.data_ptr() for a, _ in group])
            pb = (C.c_void_p * n)(*[b.data_ptr() for _, b in group])
            check(L.bin_image_metrics_batch_u8(pa, pb, n, h, w, c, flags, out[k].data_ptr(), ws.data_ptr(), ws.numel(),
                                               stream.cuda_stream))
    return out


# ----------------------------------------------------------------------------- utils/util.py:201-250
def calculate_psnr(img1, img2):
    """utils/util.py:201-208; inf when the images are equal."""
    _, s_sq, _, _, n = _metric_sums(img1, img2, "calculate_psnr")
    mse = s_sq / n                          # == np.mean of the exact squares: the sum is exact below 2^53
    if mse == 0:
        return float('inf')
    return 20 * math.log10(255.0 / math.sqrt(mse))


def calculate_ssim(img1, img2):
    """utils/util.py:234-252: the Gaussian-11 SSIM over all channels of an (h, w), (h, w, 1) or (h, w, 3) image."""
    if not img1.shape == img2.shape:
        raise ValueError(_DIMS_MSG)
    if img1.ndim not in (2, 3):
        raise ValueError('Wrong input image dimensions.')
    return np.float64(_metric_sums(img1, img2, "calculate_ssim")[2])


# ----------------------------------------------------------------------------- skimage.measure (scikit-image <= 0.17)
def _reject(fn: str, **given):
    for name, (value, default) in given.items():
        if not (value is default or value == default):
            raise BinB200Error(f"{fn}: {name}={value!r} is not supported (only the default, {default!r}, is)")


def compare_psnr(im_true, im_test, data_range=None):
    """skimage.measure.compare_psnr for uint8 images: 10*log10(255**2 / mse), inf when they are equal."""
    if data_range is not None:
        _reject("compare_psnr", data_range=(data_range, 255))
    if not im_true.shape == im_test.shape:
        raise ValueError(_DIMS_MSG)
    _, s_sq, _, _, n = _metric_sums(im_true, im_test, "compare_psnr")
    err = np.float64(s_sq / n)
    if err == 0:
        return np.float64(np.inf)
    return 10 * np.log10((255 ** 2) / err)


_SSIM_KWARGS = {"K1": 0.01, "K2": 0.03, "sigma": 1.5, "use_sample_covariance": True}


def compare_ssim(X, Y, win_size=None, gradient=False, data_range=None, multichannel=False, gaussian_weights=False,
                 full=False, **kwargs):
    """skimage.measure.compare_ssim with its defaults (7x7 uniform window, sample covariance) on uint8 images: a 2-D
    image with multichannel=False, or an (h, w, c) image with multichannel=True (the per-channel mean)."""
    fn = "compare_ssim"
    if win_size is not None:
        _reject(fn, win_size=(win_size, 7))
    if data_range is not None:
        _reject(fn, data_range=(data_range, 255))
    _reject(fn, gradient=(gradient, False), gaussian_weights=(gaussian_weights, False), full=(full, False))
    for k, v in kwargs.items():
        if k not in _SSIM_KWARGS:
            raise BinB200Error(f"{fn}: option {k}={v!r} is not supported")
        _reject(fn, **{k: (v, _SSIM_KWARGS[k])})
    if not X.shape == Y.shape:
        raise ValueError(_DIMS_MSG)
    if multichannel != (X.ndim == 3):
        raise BinB200Error(f"{fn}: multichannel={multichannel!r} with a {X.ndim}-D image is not supported "
                           "(use multichannel=True for (h, w, c) images and False for (h, w) ones)")
    return np.float64(_metric_sums(X, Y, fn)[3])


def install_skimage_measure():
    """Make ``from skimage.measure import compare_ssim, compare_psnr`` (test.py:33) resolve to the functions above.
    If skimage.measure imports, the two attributes are added to it and nothing else is touched; otherwise stub
    ``skimage`` and ``skimage.measure`` modules are registered in sys.modules.  Idempotent.  -> the measure module."""
    try:
        import skimage.measure as measure
    except ImportError:
        sk = sys.modules.get("skimage")
        if sk is None:
            sk = types.ModuleType("skimage")
            sk.__path__ = []
            sk.__doc__ = "stub registered by bin_b200.metrics.install_skimage_measure"
            sys.modules["skimage"] = sk
        measure = types.ModuleType("skimage.measure")
        measure.__doc__ = "compare_ssim / compare_psnr of scikit-image <= 0.17, computed by bin_b200 on the GPU"
        sys.modules["skimage.measure"] = measure
        sk.measure = measure
    measure.compare_ssim = compare_ssim
    measure.compare_psnr = compare_psnr
    return measure
