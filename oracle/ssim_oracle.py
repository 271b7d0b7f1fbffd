"""fp64 torch restatement of the 'cb+ssim' training criterion (DESIGN §4r) -- TEST INFRASTRUCTURE ONLY.

``ssim_map`` is the SSIM map of utils/util.py:211-231 for (B, C, H, W) tensors at data range 1: the window
outer(g, g), g = cv2.getGaussianKernel(11, 1.5), valid correlation (the reference's [5:-5, 5:-5] crop), C1 = 0.01^2 and
C2 = 0.03^2.  It is differentiable, so autograd on it gives the reference gradients.  ``oracle/make_golden_ssim.py``
runs the unmodified utils/util.py ``ssim`` on x * 255 into ``tests/golden/ssim_loss.npz``, and the CPU tests pin this
restatement to it.  SSIM is unchanged when the images and the constants scale together, so the two agree up to
rounding.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import torch

from .metrics_oracle import GAUSS11

C1 = 0.01 ** 2
C2 = 0.03 ** 2
CYCLE_PAIRS = ((1, 7), (5, 9), (2, 8))


def _filt(x: torch.Tensor) -> torch.Tensor:
    """Valid 11 x 11 correlation of every plane of (B, C, H, W) with outer(g, g), as two 1-D passes."""
    g = torch.tensor(GAUSS11, dtype=x.dtype, device=x.device)
    n, c, h, w = x.shape
    y = x.reshape(n * c, 1, h, w)
    y = torch.nn.functional.conv2d(y, g.view(1, 1, 11, 1))
    y = torch.nn.functional.conv2d(y, g.view(1, 1, 1, 11))
    return y.reshape(n, c, h - 10, w - 10)


def ssim_map(a: torch.Tensor, b: torch.Tensor, c1: float = C1, c2: float = C2) -> torch.Tensor:
    """(B, C, H - 10, W - 10): utils/util.py:220-230 per plane."""
    mu1, mu2 = _filt(a), _filt(b)
    mu1_sq, mu2_sq, mu1_mu2 = mu1 ** 2, mu2 ** 2, mu1 * mu2
    sigma1_sq = _filt(a * a) - mu1_sq
    sigma2_sq = _filt(b * b) - mu2_sq
    sigma12 = _filt(a * b) - mu1_mu2
    return ((2 * mu1_mu2 + c1) * (2 * sigma12 + c2)) / ((mu1_sq + mu2_sq + c1) * (sigma1_sq + sigma2_sq + c2))


def ssim(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """The mean over batch, channel and valid position (fp64 in, fp64 out)."""
    return ssim_map(a, b).mean()


def charbonnier(a: torch.Tensor, b: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    """models/loss.py:130-140 CharbonnierLoss: mean sqrt(d^2 + eps)."""
    return torch.sqrt((a - b) ** 2 + eps).mean()


def cb_ssim_loss(outs: Sequence[torch.Tensor], gts: Sequence[torch.Tensor], weight: float, eps: float = 1e-6,
                 cycle_pairs: Sequence[Tuple[int, int]] = CYCLE_PAIRS) -> Tuple[torch.Tensor, List[torch.Tensor]]:
    """bin_model.get_loss with every term Charbonnier + weight * (1 - SSIM): -> (mean of the terms, the terms)."""
    pairs = list(zip(outs, gts)) + [(outs[i], outs[j]) for i, j in cycle_pairs]
    terms = [charbonnier(x, y, eps) + weight * (1 - ssim(x, y)) for x, y in pairs]
    return torch.stack(terms).mean(), terms
