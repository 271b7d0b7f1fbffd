"""Thin torch-tensor wrappers over the C ABI (device pointers + current stream).

These are the unit-level entry points used by the tests and by bin_b200.rdn; none of them
computes anything in Python/PyTorch.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import Act, ConvArgs, Frames, check, lib


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _req(t: torch.Tensor, dtype, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.BinB200Error(f"{name}: expected a CUDA tensor (bin_b200 has no CPU path)")
    if t.dtype != dtype:
        raise _lib.BinB200Error(f"{name}: expected dtype {dtype}, got {t.dtype}")
    return t.contiguous()


def act_view(t: torch.Tensor) -> Act:
    """P8 tensor [B, planes, H, W, 8] fp16 -> bin_act_t."""
    assert t.dtype == torch.float16 and t.dim() == 5 and t.shape[-1] == 8 and t.is_contiguous()
    return Act(t.data_ptr(), t.shape[0], t.shape[1], t.shape[2], t.shape[3])


def empty_p8(B: int, planes: int, H: int, W: int, device) -> torch.Tensor:
    return torch.empty((B, planes, H, W, 8), dtype=torch.float16, device=device)


def nchw_to_p8(x: torch.Tensor, dst: Optional[torch.Tensor] = None, plane0: int = 0, pad_to: int = 32) -> torch.Tensor:
    x = _req(x, torch.float32, "x")
    B, Cc, H, W = x.shape
    if dst is None:
        planes = ((Cc + pad_to - 1) // pad_to * pad_to) // 8
        dst = torch.zeros((B, planes, H, W, 8), dtype=torch.float16, device=x.device)
    check(lib().bin_nchw_to_p8(x.data_ptr(), Cc, act_view(dst), plane0, _stream()))
    return dst


def p8_to_nchw(src: torch.Tensor, C_: int, plane0: int = 0) -> torch.Tensor:
    B, _, H, W, _ = src.shape
    y = torch.empty((B, C_, H, W), dtype=torch.float32, device=src.device)
    check(lib().bin_p8_to_nchw(act_view(src), plane0, C_, y.data_ptr(), _stream()))
    return y


def _req_contig(t: torch.Tensor, dtype, name: str) -> torch.Tensor:
    """Like _req but never copies: the caller stores a raw pointer, and a temporary `.contiguous()` copy would be freed
    (and its block handed to the next allocation on this stream) before the kernel that reads it is launched."""
    if not t.is_cuda:
        raise _lib.BinB200Error(f"{name}: expected a CUDA tensor (bin_b200 has no CPU path)")
    if t.dtype != dtype:
        raise _lib.BinB200Error(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise _lib.BinB200Error(f"{name}: expected a contiguous tensor (call .contiguous() and keep the result alive)")
    return t


def make_frames(calls: Sequence[Sequence[torch.Tensor]], outs: Sequence[Optional[torch.Tensor]]) -> Frames:
    """Pointer table of a batched backbone launch.  Holds raw pointers: every tensor must be contiguous and must stay
    alive until the launch that consumes the table has been enqueued."""
    fr = Frames()
    fr.ncalls = len(calls)
    fr.nframes = len(calls[0])
    fr.Bc = calls[0][0].shape[0]
    for k, frames in enumerate(calls):
        assert len(frames) == fr.nframes
        for f, t in enumerate(frames):
            fr.frame[k][f] = _req_contig(t, torch.float32, "frame").data_ptr()
        fr.out[k] = _ptr(outs[k])
    return fr


def pack_frames(calls: Sequence[Sequence[torch.Tensor]], prec: int = 0) -> torch.Tensor:
    """RDN.py:211 + 107-132: concat + space-to-depth + fp16 cast, batched over calls.  prec=1 (BIN_PREC_F32X3): (hi, lo)
    fp16 pairs, 4 hi planes then 4 lo planes per 32-channel chunk, so the result has twice the planes."""
    fr = make_frames(calls, [None] * len(calls))
    B, _, H, W = calls[0][0].shape
    cin_pad = (12 * fr.nframes + 31) // 32 * 32
    dst = empty_p8(fr.ncalls * B, cin_pad // 8 * (2 if prec else 1), H // 2, W // 2, calls[0][0].device)
    check(lib().bin_pack_frames_p(C.byref(fr), H, W, act_view(dst), prec, _stream()))
    return dst


def pack_conv_weight(w: torch.Tensor, cout_pad: int, cin_pad: int, variant: int = 0, prec: int = 0) -> torch.Tensor:
    """prec=1 (BIN_PREC_F32X3): the three-slab split pack the x3 conv reads (3x the fp16 pack's size)."""
    w = _req(w, torch.float32, "weight")
    cout, cin, k, _ = w.shape
    n = lib().bin_packed_weight_bytes(cout_pad, cin_pad, k) // 2 * (3 if prec else 1)
    out = torch.empty(n, dtype=torch.float16, device=w.device)
    check(lib().bin_pack_conv_weight_p(w.data_ptr(), cout, cin, k, cout_pad, cin_pad, variant, prec, out.data_ptr(),
                                       _stream()))
    return out


def pad_bias(b: torch.Tensor, cout_pad: int) -> torch.Tensor:
    out = torch.zeros(cout_pad, dtype=torch.float32, device=b.device)
    out[: b.numel()] = b
    return out


def conv_fwd(in0: torch.Tensor, w_packed: torch.Tensor, bias_pad: torch.Tensor, ksize: int, cout_pad: int, *,
             in0_plane0: int = 0, in0_planes: Optional[int] = None,
             in1: Optional[torch.Tensor] = None, in1_plane0: int = 0, in1_planes: int = 0,
             relu: bool = False, epilogue: int = _lib.EPI_P8,
             out: Optional[torch.Tensor] = None, out_plane0: int = 0,
             res: Optional[torch.Tensor] = None, res_plane0: int = 0,
             frames: Optional[Frames] = None, variant: int = 0, sub=None, store_planes: int = 0,
             x3: bool = False) -> None:
    """bin_conv_fwd.  x3=True runs the split-fp16 kernel: tensors hold (hi, lo) pairs (twice the planes), every plane
    offset and count stays logical, and w_packed must come from pack_conv_weight(..., prec=1)."""
    a = ConvArgs()
    a.in0 = act_view(in0)
    a.in0_plane0 = in0_plane0
    a.in0_planes = in0.shape[1] // (2 if x3 else 1) - in0_plane0 if in0_planes is None else in0_planes
    a.x3 = int(x3)
    if in1 is not None and in1_planes > 0:
        a.in1 = act_view(in1)
        a.in1_plane0, a.in1_planes = in1_plane0, in1_planes
    a.w_packed = w_packed.data_ptr()
    a.bias = bias_pad.data_ptr()
    a.ksize, a.cout_pad, a.relu, a.epilogue, a.variant = ksize, cout_pad, int(relu), epilogue, variant
    if out is not None:
        a.out = act_view(out)
        a.out_plane0 = out_plane0
    if res is not None:
        a.res = act_view(res)
        a.res_plane0 = res_plane0
    if frames is not None:
        a.fr = frames
    if sub is not None:
        a.b_begin, a.b_count, a.y_begin, a.y_count = sub
    a.store_planes = store_planes
    check(lib().bin_conv_fwd(C.byref(a), _stream()))


def rdb_tail_fwd(x: torch.Tensor, g: torch.Tensor, w_conv: torch.Tensor, b_conv: torch.Tensor, w_lff: torch.Tensor,
                 b_lff: torch.Tensor, out: torch.Tensor, *, x_plane0: int = 0, g_plane0: int = 0, out_plane0: int = 0,
                 sub=(0, 0, 0, 0)) -> None:
    """Fused conv3 + LFF + residual of one RDB (RDN.py:141-147, 162-165) on P8 tensors; see bin_rdb_tail_fwd."""
    ax, ag, ao = act_view(x), act_view(g), act_view(out)
    check(lib().bin_rdb_tail_fwd(C.byref(ax), x_plane0, C.byref(ag), g_plane0, w_conv.data_ptr(), b_conv.data_ptr(),
                                 w_lff.data_ptr(), b_lff.data_ptr(), C.byref(ao), out_plane0, *sub, _stream()))

def _flipx4(srcs: Sequence[torch.Tensor], expand: bool) -> List[torch.Tensor]:
    name = "flipx4_expand" if expand else "flipx4_mean"
    if not 1 <= len(srcs) <= _lib.BIN_FLIPX4_MAX_TENSORS:
        raise _lib.BinB200Error(f"{name}: takes 1..{_lib.BIN_FLIPX4_MAX_TENSORS} tensors, got {len(srcs)}")
    srcs = [_req(t, torch.float32, name) for t in srcs]
    shape, dev = srcs[0].shape, srcs[0].device
    if len(shape) != 4 or shape[1] != 3 or (not expand and shape[0] % 4):
        raise _lib.BinB200Error(f"{name}: expected {'(B' if expand else '(4B'},3,H,W) tensors, got {tuple(shape)}")
    if any(t.shape != shape or t.device != dev for t in srcs):
        raise _lib.BinB200Error(f"{name}: all tensors must share shape and device")
    B = shape[0] if expand else shape[0] // 4
    H, W = shape[2], shape[3]
    with torch.cuda.device(dev):
        dsts = [torch.empty((4 * B if expand else B, 3, H, W), dtype=torch.float32, device=dev) for _ in srcs]
        sp = (C.c_void_p * len(srcs))(*[t.data_ptr() for t in srcs])
        dp = (C.c_void_p * len(dsts))(*[t.data_ptr() for t in dsts])
        fn = lib().bin_flipx4_expand if expand else lib().bin_flipx4_mean
        check(fn(sp, dp, len(srcs), B, H, W, _stream()))
    return dsts


def flipx4_expand(srcs: Sequence[torch.Tensor]) -> List[torch.Tensor]:
    """Each (B,3,H,W) tensor -> (4B,3,H,W): items [oB, oB+B) are orientation o = identity, flip W, flip H, flip H and W
    of utils/test_util.py:110-132 flipx4_forward (one launch for the whole list)."""
    return _flipx4(srcs, True)


def flipx4_mean(srcs: Sequence[torch.Tensor]) -> List[torch.Tensor]:
    """Each (4B,3,H,W) tensor laid out as flipx4_expand writes it -> (B,3,H,W) =
    (((y0 + flipW(y1)) + flipH(y2)) + flipHW(y3)) / 4 in fp32, flipx4_forward's order (one launch for the whole list)."""
    return _flipx4(srcs, False)


def train_batch_u8(samples: Sequence[Tuple[Sequence[torch.Tensor], int, int, int]], h: int, w: int) -> torch.Tensor:
    """Training batch of data/BIN_dataset.py BINDataset as the DataLoader collates it, built on the device.

    samples: (frames, top, left, flip) per item; frames = the 17 contiguous uint8 CUDA (H,W,3) BGR images of the item in
    output order (6 LQs, 6 GTenh, 5 GTinp), all of one shape.  Returns one fp32 (17,B,3,h,w) tensor with
    out[f,b,c,y,x] = frames_b[f][top+y, left + (w-1-x if flip else x), 2-c] / 255, one launch per 16 items."""
    B = len(samples)
    if B < 1:
        raise _lib.BinB200Error("train_batch_u8: no samples")
    dev = samples[0][0][0].device
    if dev.type != "cuda":
        raise _lib.BinB200Error("train_batch_u8: expected CUDA frames (bin_b200 has no CPU path)")
    tab = (_lib.TrainSample * B)()
    for i, (frames, top, left, flip) in enumerate(samples):
        if len(frames) != _lib.BIN_TRAIN_FRAMES:
            raise _lib.BinB200Error(f"train_batch_u8: item {i} has {len(frames)} frames, expected 17")
        shape = frames[0].shape
        for t in frames:
            if t.device != dev or t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3 or t.shape != shape \
                    or not t.is_contiguous():
                raise _lib.BinB200Error(f"train_batch_u8: item {i}: frames must be contiguous uint8 (H,W,3) tensors of "
                                        f"one shape on {dev}")
        e = tab[i]
        for f, t in enumerate(frames):
            e.src[f] = t.data_ptr()
        e.H, e.W, e.top, e.left, e.flip = shape[0], shape[1], top, left, int(flip)
    with torch.cuda.device(dev):
        out = torch.empty((_lib.BIN_TRAIN_FRAMES, B, 3, h, w), dtype=torch.float32, device=dev)
        for b0 in range(0, B, _lib.BIN_TRAIN_MAX_BATCH):
            n = min(_lib.BIN_TRAIN_MAX_BATCH, B - b0)
            check(lib().bin_train_batch_u8(C.cast(C.byref(tab, b0 * C.sizeof(_lib.TrainSample)), C.POINTER(_lib.TrainSample)),
                                           n, h, w, out.data_ptr(), B, b0, _stream()))
    return out


def convlstm_fwd(x, w, b, state=None):
    """ConvLSTMCell.forward (RDN.py:50-95) -> (h, c)."""
    x = _req(x, torch.float32, "x")
    B, _, H, W = x.shape
    h = torch.empty_like(x)
    c = torch.empty_like(x)
    cp = hp = None
    if state is not None:
        cp, hp = (_req(t, torch.float32, "state") for t in state)
    w, b = _req(w, torch.float32, "w"), _req(b, torch.float32, "b")
    cell = _lib.LstmCell(x.data_ptr(), _ptr(cp), _ptr(hp), w.data_ptr(), b.data_ptr(), h.data_ptr(), c.data_ptr())
    check(lib().bin_convlstm_fwd(C.byref(cell), 1, B, H, W, _stream()))
    return h, c


def convlstm_group(cells: Sequence[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]) -> List[torch.Tensor]:
    """1..3 ConvLSTM cells [(x, w, b), ...] from no state (RDN.py:57-68), one (B,3,H,W) shape, in one launch -> their h;
    c is not written.  The cells of one recurrent hand-off of the window (RDN.py:451-456) run this way."""
    xs = [_req(x, torch.float32, "x") for x, _, _ in cells]
    ws = [(_req(w, torch.float32, "w"), _req(b, torch.float32, "b")) for _, w, b in cells]
    if any(x.shape != xs[0].shape for x in xs):
        raise _lib.BinB200Error("convlstm_group: the cells of one launch must share their (B,3,H,W) shape")
    hs = [torch.empty_like(x) for x in xs]
    tab = (_lib.LstmCell * len(xs))(*[_lib.LstmCell(x.data_ptr(), None, None, w.data_ptr(), b.data_ptr(), h.data_ptr(), None)
                                      for x, (w, b), h in zip(xs, ws, hs)])
    B, _, H, W = xs[0].shape
    check(lib().bin_convlstm_fwd(tab, len(xs), B, H, W, _stream()))
    return hs
