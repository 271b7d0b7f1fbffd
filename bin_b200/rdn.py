"""Drop-in mirror of the reference's ``models/archs/RDN.py`` (laomao0/BIN) on H100.

Same class names, constructor signatures, forward signatures, 14-tuple return and state_dict
schema (1 332 keys / 540 unique tensors, SURVEY.md 8b) as the reference file, so that
``models/networks.py:9-10`` (``RDN_arch.bin_stage4_lstm()``), ``bin_model.test_forward``
(``bin_model.py:379-380``), ``base_model.load_network`` (strict load, ``base_model.py:89-103``)
keep working unchanged when this module is installed in its place (see INTEGRATION.md).

The nn.Modules here only HOLD the fp32 parameters; no forward does arithmetic in PyTorch.
Every forward hands device pointers to libbin_b200.so (hand-written sm_90a kernels) through
the C ABI in include/bin_b200.h and raises if the library or a CUDA device is missing.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.init as weight_init

from . import _lib, ops
from ._lib import BinB200Error, Net, check, lib

__all__ = ["set_precision", "set_self_ensemble", "set_activation_checkpointing", "ConvLSTMCell", "pixel_reshuffle", "RDB_Conv", "RDB",
           "RDN_residual_interp_2_input",
           "RDN_residual_interp_2_1_input", "RDN_residual_interp_4_1_input", "RDN_residual_interp_5_input",
           "RDN_residual_interp_5_input_ConvLSTM_L", "bin_stage4_lstm"]


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _graphs_enabled() -> bool:
    import os
    return os.environ.get("BIN_B200_GRAPH", "1") != "0"


def _check_frames(frames: Sequence[torch.Tensor]) -> Tuple[int, int, int]:
    f0 = frames[0]
    if not f0.is_cuda:
        raise BinB200Error("bin_b200 runs on CUDA (sm_90a) only; got a CPU tensor. There is no CPU fallback.")
    B, Cc, H, W = f0.shape
    if Cc != 3 or (H % 2) or (W % 2):
        raise BinB200Error(f"frames must be (B,3,H,W) with even H,W (RDN.py:123-128); got {tuple(f0.shape)}")
    for f in frames:
        if f.shape != f0.shape or f.dtype != torch.float32 or f.device != f0.device:
            raise BinB200Error("all frames must share shape, fp32 dtype and device")
    return B, H, W


# --------------------------------------------------------------------------------------------
# reference RDN.py:9-95
# --------------------------------------------------------------------------------------------
class ConvLSTMCell(nn.Module):
    """ConvLSTM cell; parameters ``Gates.{weight(12,6,3,3),bias(12)}``; Xavier-uniform / zero bias
    (RDN.py:21-38).  forward -> (h', [c', h']) like RDN.py:50-95."""

    def __init__(self, input_size, hidden_size, forget_bias=1.0, kernel_size=3, padding=3 // 2):
        super().__init__()
        if (input_size, hidden_size, kernel_size, padding, forget_bias) != (3, 3, 3, 1, 1.0):
            raise BinB200Error("bin_b200 ConvLSTMCell supports the shipped configuration (3,3,k=3,forget_bias=1) only")
        self.input_size, self.hidden_size = input_size, hidden_size
        self.Gates = nn.Conv2d(input_size + hidden_size, 4 * hidden_size, kernel_size, padding=padding, bias=True)
        self._forget_bias = forget_bias
        weight_init.xavier_uniform_(self.Gates.weight.data)
        self.Gates.bias.data.zero_()

    def forward(self, input_, prev_state):
        if torch.is_grad_enabled() and (input_.requires_grad or self.Gates.weight.requires_grad):
            from .autograd import convlstm_apply
            return convlstm_apply(self, input_, prev_state)
        state = None if prev_state is None else (prev_state[0], prev_state[1])     # (c, h), RDN.py:71
        h, c = ops.convlstm_fwd(input_, self.Gates.weight.detach(), self.Gates.bias.detach(), state)
        return h, [c, h]


def pixel_reshuffle(input, upscale_factor):
    """Space-to-depth (RDN.py:107-132) on a CUDA fp32 tensor, channel order c*r^2 + i*r + j."""
    if upscale_factor != 2:
        raise BinB200Error("pixel_reshuffle: only upscale_factor=2 is on the BIN hot path")
    x = input.contiguous()
    B, Cc, H, W = x.shape
    # one "frame" per 3 channels so that the packer's (f*3+rgb)*4+dy*2+dx order equals c*4+i*2+j
    if Cc % 3:
        raise BinB200Error("pixel_reshuffle: channel count must be a multiple of 3")
    frames = [x[:, 3 * k:3 * k + 3].contiguous() for k in range(Cc // 3)]
    if len(frames) > _lib.BIN_MAX_FRAMES:
        raise BinB200Error("pixel_reshuffle: at most 15 channels (5 frames)")
    p8 = ops.pack_frames([frames])
    return ops.p8_to_nchw(p8, Cc * 4)


# --------------------------------------------------------------------------------------------
# reference RDN.py:135-165
# --------------------------------------------------------------------------------------------
class RDB_Conv(nn.Module):
    def __init__(self, inChannels, growRate, kSize=3):
        super().__init__()
        self.conv = nn.Sequential(nn.Conv2d(inChannels, growRate, kSize, padding=(kSize - 1) // 2, stride=1), nn.ReLU())

    def forward(self, x):
        raise BinB200Error("RDB_Conv is a parameter holder; call the enclosing RDB / backbone (fused kernels)")


class RDB(nn.Module):
    """Residual dense block, RDN.py:149-165.  Standalone forward (fp32 NCHW in/out) is the
    unit-test entry; inside a backbone the block runs through bin_backbone_fwd."""

    def __init__(self, growRate0, growRate, nConvLayers, kSize=3):
        super().__init__()
        if (growRate0, growRate, nConvLayers, kSize) != (96, 32, 4, 3):
            raise BinB200Error("bin_b200 RDB supports G0=96, G=32, C=4, k=3 (the shipped bin_stage4 configuration)")
        self.convs = nn.Sequential(*[RDB_Conv(growRate0 + c * growRate, growRate) for c in range(nConvLayers)])
        self.LFF = nn.Conv2d(growRate0 + nConvLayers * growRate, growRate0, 1, padding=0, stride=1)

    def forward(self, x):
        x = x.contiguous()
        B, Cc, h, w = x.shape
        dev = x.device
        xin = ops.nchw_to_p8(x)
        g = ops.empty_p8(B, 16, h, w, dev)
        out = ops.empty_p8(B, 12, h, w, dev)
        for c in range(4):
            conv = self.convs[c].conv[0]
            wp = ops.pack_conv_weight(conv.weight.detach(), 32, 96 + 32 * c)
            ops.conv_fwd(xin, wp, ops.pad_bias(conv.bias.detach(), 32), 3, 32, in0_planes=12, in1=g, in1_planes=4 * c,
                         relu=True, out=g, out_plane0=4 * c)
        wp = ops.pack_conv_weight(self.LFF.weight.detach(), 96, 224)
        ops.conv_fwd(xin, wp, ops.pad_bias(self.LFF.bias.detach(), 96), 1, 96, in0_planes=12, in1=g, in1_planes=16,
                     out=out, res=xin)
        return ops.p8_to_nchw(out, 96)


# --------------------------------------------------------------------------------------------
# backbones, reference RDN.py:167-334
# --------------------------------------------------------------------------------------------
class _Backbone(nn.Module):
    NFRAMES = 0

    def __init__(self, G0=64, D=6, C=4, G=32):
        super().__init__()
        if (G0, D, C, G) != (96, 12, 4, 32):
            raise BinB200Error("bin_b200 backbones support G0=96, D=12, C=4, G=32 (RDN.py:418) only")
        self.G0, self.D, self.C, self.G = G0, D, C, G
        k = 3
        self.SFENet1 = nn.Conv2d(12 * self.NFRAMES, G0, 5, padding=2, stride=1)
        self.SFENet2 = nn.Conv2d(G0, G0, k, padding=1, stride=1)
        self.RDBs = nn.ModuleList([RDB(growRate0=G0, growRate=G, nConvLayers=C) for _ in range(D)])
        self.GFF = nn.Sequential(nn.Conv2d(D * G0, G0, 1, padding=0, stride=1), nn.Conv2d(G0, G0, k, padding=1, stride=1))
        self.UPNet = nn.Sequential(nn.Conv2d(G0, 256, k, padding=1, stride=1), nn.PixelShuffle(2),
                                   nn.Conv2d(64, 3, k, padding=1, stride=1))
        self._packed: Optional[torch.Tensor] = None
        self._packed_key = None

    # -- packed weights (cached per parameter version / device) ---------------------------------
    def _conv_modules(self) -> List[nn.Conv2d]:
        """The 66 convs in nn.Module registration order (= the order of bin_backbone_pack's pointer tables)."""
        ms = [self.SFENet1, self.SFENet2]
        for blk in self.RDBs:
            ms += [rc.conv[0] for rc in blk.convs] + [blk.LFF]
        ms += [self.GFF[0], self.GFF[1], self.UPNet[0], self.UPNet[2]]
        return ms

    def _conv_params(self) -> List[torch.Tensor]:
        """[w0, b0, w1, b1, ...] read from the conv modules' attributes, NOT from self.parameters(): an
        nn.DataParallel replica (bin_model.py:42) has empty _parameters and carries its broadcast weight copies as
        plain tensor attributes (torch/nn/parallel/replicate.py), and those are the tensors a replica must run on."""
        ps: List[torch.Tensor] = []
        for m in self._conv_modules():
            ps += [m.weight, m.bias]
        if len(ps) != 2 * _lib.BIN_BACKBONE_NCONV:
            raise BinB200Error("backbone does not hold the 66 convs of RDN.py:187-208")
        return ps

    def packed_blob(self, prec: int = 0) -> torch.Tensor:
        """Packed weights for BIN_PREC_F16 (0) or BIN_PREC_F32X3 (1), cached per parameter version."""
        ps = self._conv_params()
        key = (prec, ps[0].device.index) + tuple((p.data_ptr(), p._version) for p in ps)
        if prec:
            cached = self.__dict__.get("_packed_x3")
            if cached is None or cached[0] != key:
                dev = ps[0].device
                if dev.type != "cuda":
                    raise BinB200Error("bin_b200: parameters must live on a CUDA device (call .to('cuda')); no CPU fallback")
                with torch.cuda.device(dev):
                    blob = torch.empty(lib().bin_backbone_packed_bytes_p(self.NFRAMES, prec), dtype=torch.uint8, device=dev)
                    wp = (C.c_void_p * _lib.BIN_BACKBONE_NCONV)(*[p.data_ptr() for p in ps[0::2]])
                    bp = (C.c_void_p * _lib.BIN_BACKBONE_NCONV)(*[p.data_ptr() for p in ps[1::2]])
                    check(lib().bin_backbone_pack_p(self.NFRAMES, wp, bp, blob.data_ptr(), prec, _stream()))
                self.__dict__["_packed_x3"] = cached = (key, blob)
            return cached[1]
        if self._packed is None or key != self._packed_key:
            dev = ps[0].device
            if dev.type != "cuda":
                raise BinB200Error("bin_b200: parameters must live on a CUDA device (call .to('cuda')); no CPU fallback")
            for p in ps:
                if p.dtype != torch.float32 or not p.is_contiguous():
                    raise BinB200Error("bin_b200: parameters must be contiguous fp32")
            with torch.cuda.device(dev):
                blob = torch.empty(lib().bin_backbone_packed_bytes(self.NFRAMES), dtype=torch.uint8, device=dev)
                wp = (C.c_void_p * _lib.BIN_BACKBONE_NCONV)(*[p.data_ptr() for p in ps[0::2]])
                bp = (C.c_void_p * _lib.BIN_BACKBONE_NCONV)(*[p.data_ptr() for p in ps[1::2]])
                check(lib().bin_backbone_pack(self.NFRAMES, wp, bp, blob.data_ptr(), _stream()))
            self._packed, self._packed_key = blob, key
        return self._packed

    def _forward_frames(self, *frames):
        if len(frames) != self.NFRAMES:
            raise BinB200Error(f"{type(self).__name__} takes {self.NFRAMES} frames")
        if torch.is_grad_enabled() and (any(f.requires_grad for f in frames) or self.SFENet1.weight.requires_grad):
            from .autograd import backbone_apply
            return backbone_apply(self, frames)
        frames = [f.contiguous() for f in frames]
        B, H, W = _check_frames(frames)
        dev = frames[0].device
        with torch.cuda.device(dev):
            out = torch.empty_like(frames[0])
            fr = ops.make_frames([frames], [out])
            prec = _prec_of(self)
            nbytes = lib().bin_backbone_workspace_bytes_p(self.NFRAMES, B, H, W, prec)
            ws = _workspace(dev, nbytes)
            check(lib().bin_backbone_fwd_p(self.NFRAMES, self.packed_blob(prec).data_ptr(), C.byref(fr), H, W, ws.data_ptr(),
                                           ws.numel(), prec, _stream()))
        return out


class RDN_residual_interp_2_input(_Backbone):       # RDN.py:167-222
    NFRAMES = 2

    def forward(self, B0, B1):
        return self._forward_frames(B0, B1)


class RDN_residual_interp_2_1_input(_Backbone):     # RDN.py:224-280
    NFRAMES = 3

    def forward(self, I0, I1, I2):
        return self._forward_frames(I0, I1, I2)


class RDN_residual_interp_4_1_input(_Backbone):     # RDN.py:282-334
    NFRAMES = 5

    def forward(self, B0, B1, B2, B3, B4):
        return self._forward_frames(B0, B1, B2, B3, B4)


_WS = {}
PRECISIONS = {"fp16": 0, "fp32": 1}


def _prec_of(module) -> int:
    """`module.precision` = "fp16" (default: fp16 storage / fp32 accumulate, <=1e-3) or "fp32" (split-fp16 x3 mode,
    <=1e-5, ~3x slower).  Set it on the top-level net with set_precision(); sub-modules inherit through the attribute."""
    name = getattr(module, "precision", "fp16")
    if name not in PRECISIONS:
        raise BinB200Error(f"unknown precision {name!r}; use 'fp16' or 'fp32'")
    return PRECISIONS[name]


def set_precision(net: nn.Module, precision: str) -> nn.Module:
    if precision not in PRECISIONS:
        raise BinB200Error(f"unknown precision {precision!r}; use 'fp16' or 'fp32'")
    for m in net.modules():
        m.precision = precision
    return net


CHECKPOINTING = (None, "recompute")


def _checkpointing_of(module) -> Optional[str]:
    mode = getattr(module, "activation_checkpointing", None)
    if mode not in CHECKPOINTING:
        raise BinB200Error(f"unknown activation checkpointing mode {mode!r}; use None or 'recompute'")
    return mode


def set_activation_checkpointing(net: nn.Module, mode: Optional[str]) -> nn.Module:
    """Choose what a grad-enabled forward keeps for the backward, for every module in `net.modules()` (so a DataParallel
    wrapper or a module holding the net works).  None (the default): each batched backbone stage keeps its training
    workspace, growth maps of all 12 RDBs included, until its backward.  "recompute": each stage keeps only its input
    frames; its backward re-runs the inference forward and rebuilds each RDB's growth maps, so a step holds one stage's
    activations at a time instead of all of them, at the price of extra forward work.  Every kernel sees the same
    operands in both modes: outputs, frame gradients and conv weight gradients are bit-identical, and the values that
    existing kernels sum with float atomics (loss terms, bias and ConvLSTM gradients) vary only in their last bits, as
    they do from run to run in either mode.  A plain attribute, not a parameter or buffer: the state_dict is
    unchanged."""
    if mode not in CHECKPOINTING:
        raise BinB200Error(f"unknown activation checkpointing mode {mode!r}; use None or 'recompute'")
    for m in net.modules():
        m.activation_checkpointing = mode
    return net


def _ws_key(dev: torch.device):
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    return (idx, torch.cuda.current_stream(idx).cuda_stream)


def _workspace(dev: torch.device, nbytes: int) -> torch.Tensor:
    """Grow-only scratch buffer per (device, stream) -- the C ABI never allocates, and two streams (or the worker
    threads of nn.DataParallel, one per replica device, bin_model.py:42) must never share scratch memory: launches on
    different streams are not ordered against each other.  Same-stream callers reuse one buffer (stream order)."""
    key = _ws_key(dev)
    cur = _WS.get(key)
    if cur is None or cur.numel() < nbytes:
        _WS[key] = None
        cur = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _WS[key] = cur
    return cur


def release_workspaces() -> None:
    """Drop every cached scratch buffer (they are re-created on demand)."""
    _WS.clear()


# --------------------------------------------------------------------------------------------
# temporal pyramid, reference RDN.py:337-405
# --------------------------------------------------------------------------------------------
class RDN_residual_interp_5_input(nn.Module):
    def __init__(self, lstm=False, GO=64, D=6):
        super().__init__()
        if not lstm:
            raise BinB200Error("only the lstm=True pyramid is shipped by the reference (RDN.py:355-365 needs a missing class)")
        self.lstm = lstm
        self.model1_1 = RDN_residual_interp_2_input(G0=GO, D=D)
        self.model1_2 = self.model1_1
        self.model1_3 = self.model1_1
        self.model1_4 = self.model1_1
        self.model2_1 = RDN_residual_interp_2_1_input(G0=GO, D=D)
        self.model2_2 = self.model2_1
        self.model2_3 = self.model2_1
        self.model3_1 = RDN_residual_interp_4_1_input(G0=GO, D=D)
        self.model3_2 = self.model3_1
        self.model4_1 = RDN_residual_interp_4_1_input(G0=GO, D=D)

    def forward(self, B1, B3, B5, B7, B9, previous_input=None):
        """10 backbone calls of RDN.py:367-405, issued as 4 batched launches (same-weight calls
        ride along the batch dimension)."""
        if torch.is_grad_enabled() and (any(t.requires_grad for t in (B1, B3, B5, B7, B9)) or
                                        self.model1_1.SFENet1.weight.requires_grad):
            from .autograd import pyramid_apply
            return pyramid_apply(self, B1, B3, B5, B7, B9, previous_input)
        m1, m2, m3, m4 = self.model1_1, self.model2_1, self.model3_1, self.model4_1
        I2, I4, I6, I8 = _batched(m1, [(B1, B3), (B3, B5), (B5, B7), (B7, B9)])
        if previous_input is not None and previous_input[0] is not None:
            p4, p6, p8, p5, p7, p6b = previous_input
            I3, I5, I7 = _batched(m2, [(p4, I2, I4), (p6, I4, I6), (p8, I6, I8)])
            I4b, I6b = _batched(m3, [(p5, B3, I3, I5, B5), (p7, B5, I5, I7, B7)])
            (I5c,) = _batched(m4, [(p6b, I4, I4b, I6b, I6)])
        else:
            I3, I5, I7 = _batched(m2, [(I2, I2, I4), (I4, I4, I6), (I6, I6, I8)])
            I4b, I6b = _batched(m3, [(I3, B3, I3, I5, B5), (I5, B5, I5, I7, B7)])
            (I5c,) = _batched(m4, [(I4, I4, I4b, I6b, I6)])
        return I2, I4, I6, I8, I3, I5, I7, I4b, I6b, I5c


def _batched(model: _Backbone, calls):
    calls = [[t.contiguous() for t in c] for c in calls]
    B, H, W = _check_frames([t for c in calls for t in c])
    dev = calls[0][0].device
    with torch.cuda.device(dev):
        outs = [torch.empty_like(calls[0][0]) for _ in calls]
        fr = ops.make_frames(calls, outs)
        prec = _prec_of(model)
        nbytes = lib().bin_backbone_workspace_bytes_p(model.NFRAMES, B * len(calls), H, W, prec)
        ws = _workspace(dev, nbytes)
        check(lib().bin_backbone_fwd_p(model.NFRAMES, model.packed_blob(prec).data_ptr(), C.byref(fr), H, W, ws.data_ptr(),
                                       ws.numel(), prec, _stream()))
    return outs


# --------------------------------------------------------------------------------------------
# two-step recurrent wrapper, reference RDN.py:408-465
# --------------------------------------------------------------------------------------------
_LSTM_NAMES = ["clstm_4_prime", "clstm_6_prime", "clstm_8_prime", "clstm_5_prime_prime", "clstm_7_prime_prime",
               "clstm_6_prime_prime_prime"]


class RDN_residual_interp_5_input_ConvLSTM_L(nn.Module):
    def __init__(self, modelType='lstm'):
        super().__init__()
        if modelType != 'lstm':
            raise BinB200Error("only modelType='lstm' is on the BIN hot path (RDN.py:449)")
        self.modelType = modelType
        for n in _LSTM_NAMES:                                   # RDN.py:412-417 (registration order matters)
            setattr(self, n, ConvLSTMCell(3, 3))
        self.model = RDN_residual_interp_5_input(lstm=True, GO=96, D=12)   # RDN.py:418
        self.prev_state = None
        self.hidden_state = None

    def _all_tensors(self) -> List[torch.Tensor]:
        """Every weight the window reads (4 unique backbones + 6 ConvLSTM cells), replica-safe (see _conv_params)."""
        pyr = self.model
        ts: List[torch.Tensor] = []
        for m in (pyr.model1_1, pyr.model2_1, pyr.model3_1, pyr.model4_1):
            ts += m._conv_params()
        for n in _LSTM_NAMES:
            g = getattr(self, n).Gates
            ts += [g.weight, g.bias]
        return ts

    def _net(self, prec: int = 0) -> Net:
        net = Net()
        pyr = self.model
        for k, m in enumerate((pyr.model1_1, pyr.model2_1, pyr.model3_1, pyr.model4_1)):
            net.blob[k] = m.packed_blob(prec).data_ptr()
        for k, n in enumerate(_LSTM_NAMES):
            cell = getattr(self, n)
            net.lstm_w[k] = cell.Gates.weight.data_ptr()
            net.lstm_b[k] = cell.Gates.bias.data_ptr()
        return net

    def forward(self, B1, B3, B5, B7, B9, B11):
        """One 6-frame window -> the reference's 14-tuple (RDN.py:461-465): executes 17 unique
        backbone calls of its 20 and the 6 live ConvLSTM calls of its 12 (SURVEY.md App. A)."""
        frames = [B1, B3, B5, B7, B9, B11]
        ensemble = _ensemble_of(self)
        if torch.is_grad_enabled() and (any(f.requires_grad for f in frames) or
                                        any(p.requires_grad for p in self._all_tensors())):
            if ensemble is not None:
                raise BinB200Error(f"self-ensemble {ensemble!r} is inference-only: call the net under torch.no_grad(), "
                                   "or set_self_ensemble(net, None) to train")
            from .autograd import window_apply
            return window_apply(self, frames)
        frames = [f.contiguous() for f in frames]
        B, H, W = _check_frames(frames)
        dev = frames[0].device
        if ensemble is not None:
            return self._forward_flipx4(frames, B, H, W, dev)
        if _graphs_enabled() and not getattr(self, "_is_replica", False) and not torch.cuda.is_current_stream_capturing():
            return self._forward_graphed(frames, B, H, W, dev)
        with torch.cuda.device(dev):
            return tuple(self._launch_window(frames, B, H, W, dev)[0])

    def _launch_window(self, frames, B, H, W, dev):
        outs = [torch.empty_like(frames[0]) for _ in range(14)]
        prec = _prec_of(self)
        net = self._net(prec)
        ws = _workspace(dev, lib().bin_window_workspace_bytes_p(B, H, W, prec))
        fp = (C.c_void_p * 6)(*[f.data_ptr() for f in frames])
        op = (C.c_void_p * 14)(*[o.data_ptr() for o in outs])
        check(lib().bin_window_fwd_p(C.byref(net), fp, op, B, H, W, ws.data_ptr(), ws.numel(), prec, _stream()))
        return outs, ws

    def _forward_flipx4(self, frames, B, H, W, dev):
        """x4 flip self-ensemble (utils/test_util.py:110-132 flipx4_forward, applied to all 6 frames and all 14 outputs):
        the four orientations run as ONE window at batch 4B, then each output is flipped back and averaged.  Eager, not
        graphed: a graph capture would hold a second batch-4B workspace (about 25 GB at 768x1344) in its private pool."""
        with torch.cuda.device(dev):
            big = ops.flipx4_expand(frames)
            outs, _ = self._launch_window(big, 4 * B, H, W, dev)
            del big
            return tuple(ops.flipx4_mean(outs))

    def _forward_graphed(self, frames, B, H, W, dev):
        """The ~340 kernel launches of a window are captured once per (shape, weight version) into a
        CUDA graph and replayed: removes ~10 % of host launch overhead at 720p.  Inputs are copied
        into the graph's static buffers, outputs are returned as fresh tensors (SURVEY 8b)."""
        key = (dev.index, B, H, W, _prec_of(self), tuple((p.data_ptr(), p._version) for p in self._all_tensors()))
        ent = self.__dict__.get("_graph_entry")
        with torch.cuda.device(dev):
            if ent is None or ent["key"] != key:
                self.__dict__["_graph_entry"] = None
                static_in = [torch.empty_like(f) for f in frames]
                for d, f in zip(static_in, frames):
                    d.copy_(f)
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):                       # warm-up: packs weights, opts kernels into their smem
                    self._launch_window(static_in, B, H, W, dev)
                    _WS.pop(_ws_key(dev), None)                     # the side stream's scratch buffer is not needed again
                torch.cuda.current_stream().wait_stream(side)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    static_out, ws = self._launch_window(static_in, B, H, W, dev)
                    _WS.pop(_ws_key(dev), None)                     # owned by this entry (graph-private memory pool)
                ent = {"key": key, "graph": graph, "in": static_in, "out": static_out, "ws": ws}
                self.__dict__["_graph_entry"] = ent
            else:
                for d, f in zip(ent["in"], frames):
                    d.copy_(f)
            ent["graph"].replay()
            return tuple(o.clone() for o in ent["out"])

    def forward_pyramid3(self, B1, B3, B5, B7):
        """BASELINE config 2a: stages 1-3 on 4 frames -> [I2',I4',I6',I3',I5',I4''] (SURVEY 8d)."""
        if _ensemble_of(self) is not None:
            raise BinB200Error("forward_pyramid3 has no self-ensemble mode; set_self_ensemble(net, None) first")
        if torch.is_grad_enabled() and (any(f.requires_grad for f in (B1, B3, B5, B7)) or
                                        self.model.model1_1.SFENet1.weight.requires_grad):
            from .autograd import pyramid3_apply                      # BASELINE config 3a (training on the 4-frame graph)
            return pyramid3_apply(self, (B1, B3, B5, B7))
        frames = [f.contiguous() for f in (B1, B3, B5, B7)]
        B, H, W = _check_frames(frames)
        dev = frames[0].device
        with torch.cuda.device(dev):
            outs = [torch.empty_like(frames[0]) for _ in range(6)]
            net = self._net()
            ws = _workspace(dev, lib().bin_window_workspace_bytes(B, H, W))
            fp = (C.c_void_p * 4)(*[f.data_ptr() for f in frames])
            op = (C.c_void_p * 6)(*[o.data_ptr() for o in outs])
            check(lib().bin_pyramid3_fwd(C.byref(net), fp, op, B, H, W, ws.data_ptr(), ws.numel(), _stream()))
        return tuple(outs)


def bin_stage4_lstm():
    """Factory with the reference's name and arity (RDN.py:469-471; networks.py:9-10)."""
    return RDN_residual_interp_5_input_ConvLSTM_L()


ENSEMBLES = (None, "flipx4")


def _ensemble_of(module) -> Optional[str]:
    mode = getattr(module, "self_ensemble", None)
    if mode not in ENSEMBLES:
        raise BinB200Error(f"unknown self-ensemble mode {mode!r}; use None or 'flipx4'")
    return mode


def set_self_ensemble(net: nn.Module, mode: Optional[str]) -> nn.Module:
    """Turn the x4 flip self-ensemble of utils/test_util.py:110-132 on (mode "flipx4") or off (None) for every window net
    in `net.modules()` (so a DataParallel wrapper or a model object holding the net works).  Inference only: a
    grad-enabled call then raises.  It is a plain attribute, not a parameter or buffer: the state_dict is unchanged."""
    if mode not in ENSEMBLES:
        raise BinB200Error(f"unknown self-ensemble mode {mode!r}; use None or 'flipx4'")
    nets = [m for m in net.modules() if isinstance(m, RDN_residual_interp_5_input_ConvLSTM_L)]
    if not nets:
        raise BinB200Error("set_self_ensemble: no RDN_residual_interp_5_input_ConvLSTM_L in this module")
    for m in nets:
        m.self_ensemble = mode
    return net
