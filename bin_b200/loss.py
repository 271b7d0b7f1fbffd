"""Fused pixel loss of the training step (SURVEY 8f rank 3): bin_model.get_loss, bin_model.py:395-425.

`pixel_loss(outs, gts, kind)` returns (loss, loss_list) exactly like `get_loss(ret=1)` for the shipped configuration
(nframes == 6, version == 2: 14 output-vs-GT terms + 3 cycle terms on output pairs (1,7), (5,9), (2,8), averaged over
the 17 terms).  One reduction launch and one gradient launch replace ~50 element-wise / reduce kernels."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import torch

from ._lib import BinB200Error, check, lib
from .autograd import deterministic_flags

KINDS = {"l1": 0, "l2": 1, "cb": 2}                   # bin_model.py:54-59
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
        flags = deterministic_flags()                 # torch.use_deterministic_algorithms: fixed-order sums
        with torch.cuda.device(dev):
            pair = torch.empty(npairs, device=dev)
            scratch = (torch.empty(lib().bin_pixel_loss_scratch_bytes(npairs, n), dtype=torch.uint8, device=dev)
                       if flags else None)
            ap = (C.c_void_p * npairs)(*[t.data_ptr() for t in a])
            bp = (C.c_void_p * npairs)(*[t.data_ptr() for t in b])
            check(lib().bin_pixel_loss_fwd_ex(ap, bp, npairs, n, kind, eps, pair.data_ptr(), flags,
                                              None if scratch is None else scratch.data_ptr(),
                                              0 if scratch is None else scratch.numel(), _stream()))
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
        dev = a[0].device
        with torch.cuda.device(dev):
            up = gtotal.reshape(1).float().contiguous()
            da = [torch.empty_like(t) for t in a]
            db = [torch.empty_like(t) if need else None for t, need in zip(b, ctx.need_b)]
            P = lambda ts: (C.c_void_p * npairs)(*[None if t is None else t.data_ptr() for t in ts])
            check(lib().bin_pixel_loss_bwd(P(a), P(b), P(da), P(db), npairs, ctx.n, ctx.kind, ctx.eps, up.data_ptr(), _stream()))
        return (None, None, None, *da, *db)


def pixel_loss(outs: Sequence[torch.Tensor], gts: Sequence[torch.Tensor], kind: str = "l1", eps: float = 1e-6,
               cycle_pairs: Optional[Sequence[Tuple[int, int]]] = None, nframes: Optional[int] = None,
               version: int = 2) -> Tuple[torch.Tensor, List[torch.Tensor]]:
    """`cycle_pairs` defaults to what get_loss uses for (nframes, version); nframes defaults to 6 for the shipped
    14-output graph and must be given (or cycle_pairs passed) for any other output count."""
    if cycle_pairs is None:
        if nframes is None:
            if len(outs) != 14:
                raise BinB200Error("pixel_loss: pass nframes/version (bin_model.get_info) or cycle_pairs when the graph "
                                   "does not have the shipped 14 outputs")
            nframes = 6
        cycle_pairs = cycle_pairs_for(nframes, version)
    if any(max(i, j) >= len(outs) for i, j in cycle_pairs):
        raise BinB200Error("pixel_loss: cycle pair index outside the output list")
    if kind not in KINDS:
        raise BinB200Error(f"unknown pixel criterion {kind!r} (bin_model.py:54-61 knows l1, l2, cb)")
    if len(outs) != len(gts):
        raise BinB200Error("pixel_loss: one target per output (bin_model.get_info)")
    a = list(outs) + [outs[i] for i, _ in cycle_pairs]
    b = list(gts) + [outs[j] for _, j in cycle_pairs]
    total, pair = PixelLossFn.apply(KINDS[kind], float(eps), len(a), *a, *b)
    return total, [pair[k] for k in range(len(outs))]
