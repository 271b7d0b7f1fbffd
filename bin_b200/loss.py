"""Fused pixel loss of the training step (SURVEY 8f rank 3): bin_model.get_loss, bin_model.py:395-425.

`pixel_loss(outs, gts, kind)` returns (loss, loss_list) exactly like `get_loss(ret=1)` for the shipped configuration
(nframes == 6, version == 2: 14 output-vs-GT terms + 3 cycle terms on output pairs (1,7), (5,9), (2,8), averaged over
the 17 terms).  One reduction launch and one gradient launch replace ~50 element-wise / reduce kernels.

`pixel_loss(outs, gts, "cb+ssim", ssim_weight=w)` makes each term Charbonnier(a, b) + w * (1 - SSIM(a, b)) (DESIGN
§4r): the `cb` launches, then one SSIM launch over all terms (ssim_loss.cu).  `ssim(a, b)` is the differentiable mean
SSIM of one pair."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import torch

from ._lib import BinB200Error, check, lib
from .autograd import deterministic_flags

KINDS = {"l1": 0, "l2": 1, "cb": 2}                   # bin_model.py:54-59
CB_SSIM = "cb+ssim"                                   # Charbonnier + ssim_weight * (1 - SSIM), DESIGN §4r
CYCLE_PAIRS_6V2 = ((1, 7), (5, 9), (2, 8))            # bin_model.py:409-416
CYCLE_PAIRS_4V5 = ((1, 5),)                           # bin_model.py:405-408


def cycle_pairs_for(nframes: int, version: int) -> Tuple[Tuple[int, int], ...]:
    """The cycle terms bin_model.get_loss appends for a (nframes, version) configuration (bin_model.py:405-416)."""
    if nframes == 6 and version == 2:
        return CYCLE_PAIRS_6V2
    if nframes == 4 and version == 5:
        return CYCLE_PAIRS_4V5
    return ()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptrs(ts) -> C.Array:
    return (C.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])


def _pair_fwd(kind: int, eps: float, a: List[torch.Tensor], b: List[torch.Tensor]) -> torch.Tensor:
    """One bin_pixel_loss_fwd_ex launch: -> cri_pix(a_k, b_k) per pair (fp32[npairs] on the device)."""
    npairs, n, dev = len(a), a[0].numel(), a[0].device
    flags = deterministic_flags()                 # torch.use_deterministic_algorithms: fixed-order sums
    with torch.cuda.device(dev):
        pair = torch.empty(npairs, device=dev)
        scratch = (torch.empty(lib().bin_pixel_loss_scratch_bytes(npairs, n), dtype=torch.uint8, device=dev)
                   if flags else None)
        check(lib().bin_pixel_loss_fwd_ex(_ptrs(a), _ptrs(b), npairs, n, kind, eps, pair.data_ptr(), flags,
                                          None if scratch is None else scratch.data_ptr(),
                                          0 if scratch is None else scratch.numel(), _stream()))
    return pair


def _pair_bwd(kind: int, eps: float, a, b, need_b, gtotal: torch.Tensor):
    """One bin_pixel_loss_bwd launch: -> (da, db) per pair, written (db[k] is None where need_b[k] is False)."""
    npairs, dev = len(a), a[0].device
    with torch.cuda.device(dev):
        up = gtotal.reshape(1).float().contiguous()
        da = [torch.empty_like(t) for t in a]
        db = [torch.empty_like(t) if need else None for t, need in zip(b, need_b)]
        check(lib().bin_pixel_loss_bwd(_ptrs(a), _ptrs(b), _ptrs(da), _ptrs(db), npairs, a[0].numel(), kind, eps,
                                       up.data_ptr(), _stream()))
    return da, db


class PixelLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, kind: int, eps: float, npairs: int, *tensors):
        a = [t.detach().contiguous().float() for t in tensors[:npairs]]
        b = [t.detach().contiguous().float() for t in tensors[npairs:]]
        n = a[0].numel()
        dev = a[0].device
        if not a[0].is_cuda:
            raise BinB200Error("bin_b200.loss runs on CUDA tensors only (no CPU fallback)")
        if any(t.numel() != n or t.device != dev for t in a + b):
            raise BinB200Error("pixel_loss: all tensors must share size and device")
        pair = _pair_fwd(kind, eps, a, b)
        ctx.kind, ctx.eps, ctx.npairs, ctx.n = kind, eps, npairs, n
        ctx.need_b = [t.requires_grad for t in tensors[npairs:]]
        ctx.save_for_backward(*a, *b)
        ctx.mark_non_differentiable(pair)
        return pair.sum() / npairs, pair

    @staticmethod
    def backward(ctx, gtotal, _gpair):
        npairs = ctx.npairs
        saved = ctx.saved_tensors
        a, b = saved[:npairs], saved[npairs:]
        da, db = _pair_bwd(ctx.kind, ctx.eps, a, b, ctx.need_b, gtotal)
        return (None, None, None, *da, *db)


def pixel_loss(outs: Sequence[torch.Tensor], gts: Sequence[torch.Tensor], kind: str = "l1", eps: float = 1e-6,
               cycle_pairs: Optional[Sequence[Tuple[int, int]]] = None, nframes: Optional[int] = None,
               version: int = 2, ssim_weight: Optional[float] = None) -> Tuple[torch.Tensor, List[torch.Tensor]]:
    """`cycle_pairs` defaults to what get_loss uses for (nframes, version); nframes defaults to 6 for the shipped
    14-output graph and must be given (or cycle_pairs passed) for any other output count.  kind 'cb+ssim' needs
    `ssim_weight` (the yml's train.ssim_weight); the other kinds ignore it."""
    if cycle_pairs is None:
        if nframes is None:
            if len(outs) != 14:
                raise BinB200Error("pixel_loss: pass nframes/version (bin_model.get_info) or cycle_pairs when the graph "
                                   "does not have the shipped 14 outputs")
            nframes = 6
        cycle_pairs = cycle_pairs_for(nframes, version)
    if any(max(i, j) >= len(outs) for i, j in cycle_pairs):
        raise BinB200Error("pixel_loss: cycle pair index outside the output list")
    if kind == CB_SSIM:
        total, terms, _ = pixel_ssim_loss(outs, gts, ssim_weight, eps, cycle_pairs)
        return total, terms
    if kind not in KINDS:
        raise BinB200Error(f"unknown pixel criterion {kind!r} (bin_model.py:54-61 knows l1, l2, cb; this package adds "
                           f"{CB_SSIM})")
    if len(outs) != len(gts):
        raise BinB200Error("pixel_loss: one target per output (bin_model.get_info)")
    a = list(outs) + [outs[i] for i, _ in cycle_pairs]
    b = list(gts) + [outs[j] for _, j in cycle_pairs]
    total, pair = PixelLossFn.apply(KINDS[kind], float(eps), len(a), *a, *b)
    return total, [pair[k] for k in range(len(outs))]


# ----------------------------------------------------------------------------- SSIM (DESIGN §4r)
def ssim_planes(t: torch.Tensor) -> Tuple[int, int, int]:
    """(planes, h, w) of a (B, C, H, W) tensor for the SSIM launches; H and W below 11 leave no valid position of the
    11 x 11 window and are refused."""
    if t.dim() != 4:
        raise BinB200Error(f"ssim: expected a (B, C, H, W) tensor, got shape {tuple(t.shape)}")
    n, c, h, w = t.shape
    if h < 11 or w < 11:
        raise BinB200Error(f"ssim: H and W must be at least 11 (the 11x11 window has no valid position in {h}x{w})")
    return n * c, h, w


def _ssim_fwd(a, b, keep_maps: bool):
    """One bin_ssim_loss_fwd launch: -> (SSIM sum per pair, fp32[npairs]; the backward's maps or None)."""
    npairs, dev = len(a), a[0].device
    planes, h, w = ssim_planes(a[0])
    flags = deterministic_flags()
    with torch.cuda.device(dev):
        sums = torch.empty(npairs, device=dev)
        maps = (torch.empty(lib().bin_ssim_loss_maps_bytes(npairs, planes, h, w) // 4, device=dev)
                if keep_maps else None)
        scratch = (torch.empty(lib().bin_ssim_loss_scratch_bytes(npairs, planes, h, w), dtype=torch.uint8, device=dev)
                   if flags else None)
        check(lib().bin_ssim_loss_fwd(_ptrs(a), _ptrs(b), npairs, planes, h, w, sums.data_ptr(),
                                      None if maps is None else maps.data_ptr(), flags,
                                      None if scratch is None else scratch.data_ptr(),
                                      0 if scratch is None else scratch.numel(), _stream()))
    return sums, maps


def _ssim_bwd(a, b, maps: torch.Tensor, da, db, upstream: torch.Tensor) -> None:
    """One bin_ssim_loss_bwd launch: da[k] += upstream[k] * dSum_k/da_k (and db where it is not None)."""
    planes, h, w = ssim_planes(a[0])
    with torch.cuda.device(a[0].device):
        up = upstream.float().contiguous()
        check(lib().bin_ssim_loss_bwd(_ptrs(a), _ptrs(b), maps.data_ptr(), _ptrs(da), _ptrs(db), len(a), planes, h, w,
                                      up.data_ptr(), _stream()))


def _pairs_of(tensors: Sequence[torch.Tensor], npairs: int):
    a = [t.detach().contiguous().float() for t in tensors[:npairs]]
    b = [t.detach().contiguous().float() for t in tensors[npairs:]]
    if not a[0].is_cuda:
        raise BinB200Error("bin_b200.loss runs on CUDA tensors only (no CPU fallback)")
    if any(t.shape != a[0].shape or t.device != a[0].device for t in a + b):
        raise BinB200Error("ssim: all tensors must share shape and device")
    return a, b


def _grad_wanted(tensors) -> bool:
    """Whether autograd will run the backward: the forward then keeps the SSIM maps (needs_input_grad does not see
    torch.no_grad)."""
    return torch.is_grad_enabled() and any(t.requires_grad for t in tensors)


class SsimFn(torch.autograd.Function):
    """(keep_maps, npairs, *a, *b) -> the SSIM sum of each pair, fp32[npairs]."""

    @staticmethod
    def forward(ctx, keep_maps: bool, npairs: int, *tensors):
        a, b = _pairs_of(tensors, npairs)
        sums, maps = _ssim_fwd(a, b, keep_maps)
        ctx.npairs, ctx.maps = npairs, maps
        ctx.need_b = [t.requires_grad for t in tensors[npairs:]]
        ctx.save_for_backward(*a, *b)
        return sums

    @staticmethod
    def backward(ctx, gsums):
        saved = ctx.saved_tensors
        a, b = saved[:ctx.npairs], saved[ctx.npairs:]
        da = [torch.zeros_like(t) for t in a]
        db = [torch.zeros_like(t) if need else None for t, need in zip(b, ctx.need_b)]
        _ssim_bwd(a, b, ctx.maps, da, db, gsums)
        return (None, None, *da, *db)


def ssim(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """The mean SSIM of two fp32 (B, C, H, W) CUDA tensors as a differentiable 0-d tensor: the SSIM map of
    utils/util.py:211-231 (Gaussian 11 x 11 window, sigma 1.5, valid positions only) for data range 1 (C1 = 0.01^2,
    C2 = 0.03^2), averaged over the batch, the channels and the (H - 10)(W - 10) positions.  Not clamped."""
    planes, h, w = ssim_planes(a)
    if tuple(b.shape) != tuple(a.shape):
        raise BinB200Error(f"ssim: shapes differ ({tuple(a.shape)} vs {tuple(b.shape)})")
    return SsimFn.apply(_grad_wanted((a, b)), 1, a, b)[0] / float(planes * (h - 10) * (w - 10))


class PixelSsimLossFn(torch.autograd.Function):
    """(keep_maps, eps, ssim_weight, npairs, *a, *b) -> (mean term, term per pair, mean SSIM per pair) with term =
    Charbonnier(a, b) + ssim_weight * (1 - SSIM(a, b)).  The backward's Charbonnier launch writes da / db, and the SSIM
    launch then adds to the same buffers: one fixed order."""

    @staticmethod
    def forward(ctx, keep_maps: bool, eps: float, weight: float, npairs: int, *tensors):
        a, b = _pairs_of(tensors, npairs)
        planes, h, w = ssim_planes(a[0])
        cb = _pair_fwd(KINDS["cb"], eps, a, b)
        sums, maps = _ssim_fwd(a, b, keep_maps)
        mean = sums / float(planes * (h - 10) * (w - 10))
        term = cb + weight * (1.0 - mean)
        ctx.eps, ctx.weight, ctx.npairs, ctx.maps = eps, weight, npairs, maps
        ctx.scale = -weight / (npairs * planes * (h - 10) * (w - 10))       # d total / d (SSIM sum of a pair)
        ctx.need_b = [t.requires_grad for t in tensors[npairs:]]
        ctx.save_for_backward(*a, *b)
        ctx.mark_non_differentiable(term, mean)
        return term.sum() / npairs, term, mean

    @staticmethod
    def backward(ctx, gtotal, _gterm, _gmean):
        npairs = ctx.npairs
        saved = ctx.saved_tensors
        a, b = saved[:npairs], saved[npairs:]
        da, db = _pair_bwd(KINDS["cb"], ctx.eps, a, b, ctx.need_b, gtotal)
        up = (gtotal.reshape(1).float() * ctx.scale).expand(npairs)
        _ssim_bwd(a, b, ctx.maps, da, db, up)
        return (None, None, None, None, *da, *db)


def pixel_ssim_loss(outs: Sequence[torch.Tensor], gts: Sequence[torch.Tensor], ssim_weight: Optional[float],
                    eps: float = 1e-6, cycle_pairs: Sequence[Tuple[int, int]] = CYCLE_PAIRS_6V2
                    ) -> Tuple[torch.Tensor, List[torch.Tensor], List[torch.Tensor]]:
    """The 'cb+ssim' criterion over the output-vs-GT terms and the cycle terms: -> (loss, the per-output totals, the
    per-output mean SSIM), all on the device.  pixel_loss(..., 'cb+ssim') returns the first two."""
    if ssim_weight is None:
        raise BinB200Error(f"pixel_loss: {CB_SSIM!r} needs ssim_weight")
    if len(outs) != len(gts):
        raise BinB200Error("pixel_loss: one target per output (bin_model.get_info)")
    for t in list(outs) + list(gts):
        ssim_planes(t)
    a = list(outs) + [outs[i] for i, _ in cycle_pairs]
    b = list(gts) + [outs[j] for _, j in cycle_pairs]
    total, term, mean = PixelSsimLossFn.apply(_grad_wanted(a + b), float(eps), float(ssim_weight), len(a), *a, *b)
    return total, [term[k] for k in range(len(outs))], [mean[k] for k in range(len(outs))]
