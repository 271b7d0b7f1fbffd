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
from ._lib import BinB200Error, check, lib

__all__ = ["set_precision", "set_self_ensemble", "set_activation_checkpointing", "set_outputs", "ConvLSTMCell", "pixel_reshuffle", "RDB_Conv", "RDB",
           "RDN_residual_interp_2_input",
           "RDN_residual_interp_2_1_input", "RDN_residual_interp_4_1_input", "RDN_residual_interp_5_input",
           "RDN_residual_interp_5_input_ConvLSTM_L", "bin_stage4_lstm"]


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


def _needs_grad(tensors) -> bool:
    """Whether a call takes the autograd path: grad mode is on and some tensor it reads (frames, states, any weight)
    requires a gradient.  Every tensor counts: a net whose first layer alone is frozen must still train the rest."""
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


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
        state_ts = () if prev_state is None else (prev_state[0], prev_state[1])
        if _needs_grad((input_, self.Gates.weight, self.Gates.bias) + state_ts):
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


G0_CHOICES = (64, 96)    # the widths the reference builds: 64 by default (RDN.py:171), 96 in bin_stage4_lstm (:418)
D_MAX = 12               # the shipped depth; the library's tables, masks and workspaces are sized for it


def _check_arch(G0, D, C, G) -> None:
    if G0 not in G0_CHOICES or not (isinstance(D, int) and 1 <= D <= D_MAX) or C != 4 or G != 32:
        raise BinB200Error(f"bin_b200 backbones support G0 in {G0_CHOICES}, 1 <= D <= {D_MAX}, C=4, G=32 (the "
                           f"configurations of RDN.py); got G0={G0}, D={D}, C={C}, G={G}")


class RDB(nn.Module):
    """Residual dense block, RDN.py:149-165.  Standalone forward (fp32 NCHW in/out) is the
    unit-test entry; inside a backbone the block runs through bin_backbone_fwd."""

    def __init__(self, growRate0, growRate, nConvLayers, kSize=3):
        super().__init__()
        if growRate0 not in G0_CHOICES or (growRate, nConvLayers, kSize) != (32, 4, 3):
            raise BinB200Error(f"bin_b200 RDB supports G0 in {G0_CHOICES}, G=32, C=4, k=3 (the configurations of RDN.py)")
        self.G0 = growRate0
        self.convs = nn.Sequential(*[RDB_Conv(growRate0 + c * growRate, growRate) for c in range(nConvLayers)])
        self.LFF = nn.Conv2d(growRate0 + nConvLayers * growRate, growRate0, 1, padding=0, stride=1)

    def forward(self, x):
        x = x.contiguous()
        B, Cc, h, w = x.shape
        dev = x.device
        G0, P = self.G0, self.G0 // 8
        xin = ops.nchw_to_p8(x)
        g = ops.empty_p8(B, 16, h, w, dev)
        out = ops.empty_p8(B, P, h, w, dev)
        for c in range(4):
            conv = self.convs[c].conv[0]
            wp = ops.pack_conv_weight(conv.weight.detach(), 32, G0 + 32 * c)
            ops.conv_fwd(xin, wp, ops.pad_bias(conv.bias.detach(), 32), 3, 32, in0_planes=P, in1=g, in1_planes=4 * c,
                         relu=True, out=g, out_plane0=4 * c)
        wp = ops.pack_conv_weight(self.LFF.weight.detach(), G0, G0 + 128)
        ops.conv_fwd(xin, wp, ops.pad_bias(self.LFF.bias.detach(), G0), 1, G0, in0_planes=P, in1=g, in1_planes=16,
                     out=out, res=xin)
        return ops.p8_to_nchw(out, G0)


# --------------------------------------------------------------------------------------------
# backbones, reference RDN.py:167-334
# --------------------------------------------------------------------------------------------
class _Backbone(nn.Module):
    NFRAMES = 0

    def __init__(self, G0=64, D=6, C=4, G=32):
        super().__init__()
        _check_arch(G0, D, C, G)
        self.G0, self.D, self.C, self.G = G0, D, C, G
        k = 3
        self.SFENet1 = nn.Conv2d(12 * self.NFRAMES, G0, 5, padding=2, stride=1)
        self.SFENet2 = nn.Conv2d(G0, G0, k, padding=1, stride=1)
        self.RDBs = nn.ModuleList([RDB(growRate0=G0, growRate=G, nConvLayers=C) for _ in range(D)])
        self.GFF = nn.Sequential(nn.Conv2d(D * G0, G0, 1, padding=0, stride=1), nn.Conv2d(G0, G0, k, padding=1, stride=1))
        self.UPNet = nn.Sequential(nn.Conv2d(G0, 256, k, padding=1, stride=1), nn.PixelShuffle(2),
                                   nn.Conv2d(64, 3, k, padding=1, stride=1))

    @property
    def arch(self) -> int:
        """The `arch` argument of the library's backbone calls (BIN_BACKBONE_ARCH): the frame count alone for the shipped
        G0 = 96, D = 12."""
        if (self.G0, self.D) == (96, 12):
            return self.NFRAMES
        return _lib.backbone_arch(self.NFRAMES, self.G0, self.D)

    @property
    def nconv(self) -> int:
        """Convs of this backbone, 5 D + 6 (66 for the shipped one)."""
        return 5 * self.D + 6

    # -- packed weights (cached per parameter version / device) ---------------------------------
    def _conv_modules(self) -> List[nn.Conv2d]:
        """The 5 D + 6 convs in nn.Module registration order (= the order of bin_backbone_pack's pointer tables)."""
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
        if len(ps) != 2 * self.nconv:
            raise BinB200Error(f"backbone does not hold the {self.nconv} convs of RDN.py:187-208")
        return ps

    def packed_blob(self, prec: int = 0) -> torch.Tensor:
        """Packed weights for BIN_PREC_F16 (0) or BIN_PREC_F32X3 (1), cached per parameter version."""
        return self._cached_pack("x3" if prec else "f16")

    def _cached_pack(self, kind: str) -> torch.Tensor:
        """Packed weights of one kind, cached per device and parameter version: "f16" and "x3" feed the forward in
        BIN_PREC_F16 and BIN_PREC_F32X3, "t" (transposed, tap-flipped) the backward's data gradients.  Each kind is its
        own __dict__ slot, assigned whole: replicate() gives an nn.DataParallel replica a shallow copy of the master's
        __dict__, so a replica packing its own weights (in its own worker thread) never writes into the master's cache."""
        ps = self._conv_params()
        key = (kind, ps[0].device.index) + tuple((p.data_ptr(), p._version) for p in ps)
        slot = "_pack_" + kind
        cached = self.__dict__.get(slot)
        if cached is not None and cached[0] == key:
            return cached[1]
        dev = ps[0].device
        if dev.type != "cuda":
            raise BinB200Error("bin_b200: parameters must live on a CUDA device (call .to('cuda')); no CPU fallback")
        for p in ps:
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise BinB200Error("bin_b200: parameters must be contiguous fp32")
        n, L = self.arch, lib()
        wp = (C.c_void_p * self.nconv)(*[p.data_ptr() for p in ps[0::2]])
        bp = (C.c_void_p * self.nconv)(*[p.data_ptr() for p in ps[1::2]])
        with torch.cuda.device(dev):
            if kind == "t":
                blob = torch.empty(L.bin_backbone_packed_t_bytes(n), dtype=torch.uint8, device=dev)
                check(L.bin_backbone_pack_t(n, wp, blob.data_ptr(), ops._stream()))
            elif kind == "x3":
                blob = torch.empty(L.bin_backbone_packed_bytes_p(n, 1), dtype=torch.uint8, device=dev)
                check(L.bin_backbone_pack_p(n, wp, bp, blob.data_ptr(), 1, ops._stream()))
            else:
                blob = torch.empty(L.bin_backbone_packed_bytes(n), dtype=torch.uint8, device=dev)
                check(L.bin_backbone_pack(n, wp, bp, blob.data_ptr(), ops._stream()))
        self.__dict__[slot] = (key, blob)
        return blob

    def _forward_frames(self, *frames):
        if len(frames) != self.NFRAMES:
            raise BinB200Error(f"{type(self).__name__} takes {self.NFRAMES} frames")
        if _needs_grad(list(frames) + self._conv_params()):
            from .autograd import backbone_apply
            return backbone_apply(self, frames)
        return _batched(self, [frames])[0]


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
    workspace, growth maps of all its RDBs included, until its backward.  "recompute": each stage keeps only its input
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
        prev = list(previous_input) if previous_input is not None and previous_input[0] is not None else []
        if _needs_grad([B1, B3, B5, B7, B9] + prev + [p for m in (self.model1_1, self.model2_1, self.model3_1,
                                                                   self.model4_1) for p in m._conv_params()]):
            from .autograd import pyramid_apply
            return pyramid_apply(self, B1, B3, B5, B7, B9, previous_input)
        return _pyramid_schedule(_batched, self, B1, B3, B5, B7, B9, previous_input)


def _pyramid_schedule(stage, pyr, B1, B3, B5, B7, B9, previous_input):
    """The 10 backbone calls of RDN.py:367-405 as 4 batched stages; stage(model, calls) runs one and returns its outputs.
    Without previous_input (the first step) the recurrent inputs p4, p6, p8, p5, p7, p6b are this step's own
    I2, I4, I6, I3, I5, I4."""
    m1, m2, m3, m4 = pyr.model1_1, pyr.model2_1, pyr.model3_1, pyr.model4_1
    first = previous_input is None or previous_input[0] is None
    I2, I4, I6, I8 = stage(m1, [(B1, B3), (B3, B5), (B5, B7), (B7, B9)])
    p4, p6, p8, p5, p7, p6b = (I2, I4, I6, None, None, I4) if first else previous_input
    I3, I5, I7 = stage(m2, [(p4, I2, I4), (p6, I4, I6), (p8, I6, I8)])
    if first:
        p5, p7 = I3, I5
    I4b, I6b = stage(m3, [(p5, B3, I3, I5, B5), (p7, B5, I5, I7, B7)])
    (I5c,) = stage(m4, [(p6b, I4, I4b, I6b, I6)])
    return I2, I4, I6, I8, I3, I5, I7, I4b, I6b, I5c


def _pyramid3_schedule(stage, pyr, F):
    """BASELINE config 2a: stages 1-3 of the pyramid on the 4 frames F (pattern of RDN.py:383-387) as 3 batched stages
    -> [I2', I4', I6', I3', I5', I4''] (SURVEY 8d); stage(model, calls) runs one and returns its outputs."""
    o0, o1, o2 = stage(pyr.model1_1, [(F[0], F[1]), (F[1], F[2]), (F[2], F[3])])
    o3, o4 = stage(pyr.model2_1, [(o0, o0, o1), (o1, o1, o2)])
    (o5,) = stage(pyr.model3_1, [(o3, F[1], o3, o4, F[2])])
    return o0, o1, o2, o3, o4, o5


def _launch_stage(model: _Backbone, calls, outs, prec: int) -> torch.Tensor:
    """One batched backbone stage (same-weight calls riding along the batch) in precision `prec`, on the current device,
    into the shared per-(device, stream) workspace, which it returns: a recomputing backward reads what it left there."""
    B, _, H, W = calls[0][0].shape
    fr = ops.make_frames(calls, outs)
    ws = _workspace(calls[0][0].device, lib().bin_backbone_workspace_bytes_p(model.arch, B * len(calls), H, W, prec))
    check(lib().bin_backbone_fwd_p(model.arch, model.packed_blob(prec).data_ptr(), C.byref(fr), H, W, ws.data_ptr(),
                                   ws.numel(), prec, ops._stream()))
    return ws


def _batched(model: _Backbone, calls, prec: Optional[int] = None):
    """Inference of one batched stage in precision `prec`, by default the net's (set_precision)."""
    calls = [[t.contiguous() for t in c] for c in calls]
    _check_frames([t for c in calls for t in c])
    with torch.cuda.device(calls[0][0].device):
        outs = [torch.empty_like(calls[0][0]) for _ in calls]
        _launch_stage(model, calls, outs, _prec_of(model) if prec is None else prec)
    return outs


# --------------------------------------------------------------------------------------------
# two-step recurrent wrapper, reference RDN.py:408-465
# --------------------------------------------------------------------------------------------
_LSTM_NAMES = ["clstm_4_prime", "clstm_6_prime", "clstm_8_prime", "clstm_5_prime_prime", "clstm_7_prime_prime",
               "clstm_6_prime_prime_prime"]


def _window_schedule(stage, lstm, pyr, F, s1, live=None):
    """Stages 2-4 of the six-frame window (RDN.py:422-465) -> the 14-tuple: the unique backbone calls of both
    recurrent steps and the 6 live ConvLSTM calls, in issue order (SURVEY App. A).  stage(model, calls) runs one
    batched backbone stage and returns its outputs; lstm(group) runs the cells of one recurrent hand-off, a list of
    (k, x) for ConvLSTM cell k (the order of _LSTM_NAMES) on input x from no state, and returns their h in that order;
    s1 holds the stage-1 outputs o[0..3], o[10] of the frame pairs.  With `live` (a node set from _window_live) only
    the calls and cells in it run, each stage with its shortened call list and each hand-off with its live cells (none
    left: lstm is not called), and every other result, s1 entries included, is None."""
    m2, m3, m4 = pyr.model2_1, pyr.model3_1, pyr.model4_1

    def run(n, model, calls):
        keep = [i for i in range(len(calls)) if live is None or (n, i) in live]
        outs = [None] * len(calls)
        if keep:
            for i, out in zip(keep, stage(model, [calls[i] for i in keep])):
                outs[i] = out
        return outs

    def cells(*group):
        todo = [(k, x) for k, x in group if live is None or ("lstm", k) in live]
        hs = dict(zip([k for k, _ in todo], lstm(todo) if todo else []))
        return [hs.get(k) for k, _ in group]

    o = [None] * 14
    o[0], o[1], o[2], o[3], o[10] = s1
    p4, p6, p8 = cells((0, o[1]), (1, o[2]), (2, o[3]))
    o[4], o[5], o[6], t0, t1, o[11] = run(2, m2, [(o[0], o[0], o[1]), (o[1], o[1], o[2]), (o[2], o[2], o[3]),
                                                  (p4, o[1], o[2]), (p6, o[2], o[3]), (p8, o[3], o[10])])
    del p4, p6, p8                      # no later call reads them: in inference their memory serves the next images
    p5, p7 = cells((3, o[5]), (4, o[6]))
    o[7], o[8], t2, o[12] = run(3, m3, [(o[4], F[1], o[4], o[5], F[2]), (o[5], F[2], o[5], o[6], F[3]),
                                        (p5, F[2], t0, t1, F[3]), (p7, F[3], t1, o[11], F[4])])
    del p5, p7, t0, t1
    (p6b,) = cells((5, o[8]))
    o[9], o[13] = run(4, m4, [(o[1], o[1], o[7], o[8], o[2]), (p6b, o[2], t2, o[12], o[3])])
    return tuple(o)


def _record_window():
    """The window's dependency graph, read off _window_schedule itself: the schedule runs on symbolic nodes, named
    (stage, position in the stage's full call list) for a backbone call and ("lstm", k) for a ConvLSTM image.
    -> (the node of each of the 14 outputs, {node: the nodes it reads})."""
    from types import SimpleNamespace
    reads = {(1, i): set() for i in range(5)}

    def stage(n, calls):
        for i, call in enumerate(calls):
            reads[(n, i)] = {x for x in call if x is not None}
        return [(n, i) for i in range(len(calls))]

    def lstm(group):
        for k, x in group:
            reads[("lstm", k)] = {x}
        return [("lstm", k) for k, _ in group]

    outs = _window_schedule(stage, lstm, SimpleNamespace(model2_1=2, model3_1=3, model4_1=4), [None] * 6, list(reads))
    return outs, reads


_OUT_NODE, _NODE_READS = _record_window()


def _window_live(wanted) -> frozenset:
    """Every node (see _record_window) a window must compute so that the outputs `wanted` (indices 0..13) come out: the
    backward closure of their nodes over the schedule's own dataflow."""
    live, todo = set(), [_OUT_NODE[i] for i in wanted]
    while todo:
        n = todo.pop()
        if n not in live:
            live.add(n)
            todo += _NODE_READS[n]
    return frozenset(live)


def _window_fwd(net, F, live, s1=None, keys=range(5)) -> tuple:
    """Inference of the window's nodes `live` (a set from _window_live) on the six contiguous frames F -> the 14 outputs,
    None where not computed.  s1: the stage-1 outputs a caller already holds (the streaming cache), None where it has
    none; the live stage-1 pairs without one run as one batched stage.  keys: a name for the frame pair of each of the
    five stage-1 positions; positions whose pairs share a name run once and share the output (an edge window of
    stream_video reads the pair of frames 0, 0 twice).  Stages 2-4 follow _window_schedule, every stage in the net's
    precision, and the live cells of each recurrent hand-off run as one ConvLSTM launch."""
    pyr = net.model
    s1 = [None] * 5 if s1 is None else list(s1)
    at = {}                                             # pair name -> the positions it fills
    for a in range(5):
        if (1, a) in live and s1[a] is None:
            at.setdefault(keys[a], []).append(a)
    need = [pos[0] for pos in at.values()]
    B, _, H, W = F[0].shape
    prec = _prec_of(net)
    with torch.cuda.device(F[0].device):
        # the shared workspace grows once, to the largest stage, before the first stage runs (also inside a graph capture)
        ncalls = [(pyr.model1_1, len(need))] + [(m, sum(1 for n in live if n[0] == st))
                                                 for st, m in ((2, pyr.model2_1), (3, pyr.model3_1), (4, pyr.model4_1))]
        _workspace(F[0].device, max([lib().bin_backbone_workspace_bytes_p(m.arch, B * k, H, W, prec)
                                     for m, k in ncalls if k], default=0))
        stage = lambda model, calls: _batched(model, calls, prec)
        if need:
            for pos, out in zip(at.values(), stage(pyr.model1_1, [(F[a], F[a + 1]) for a in need])):
                for a in pos:
                    s1[a] = out
        gates = [getattr(net, n).Gates for n in _LSTM_NAMES]
        lstm = lambda group: ops.convlstm_group([(x, gates[k].weight.detach(), gates[k].bias.detach()) for k, x in group])
        return _window_schedule(stage, lstm, pyr, F, s1, live)


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

    def forward(self, B1, B3, B5, B7, B9, B11):
        """One 6-frame window -> the reference's 14-tuple (RDN.py:461-465): executes 17 unique
        backbone calls of its 20 and the 6 live ConvLSTM calls of its 12 (SURVEY.md App. A), or, with set_outputs,
        only the calls the wanted outputs depend on."""
        frames = [B1, B3, B5, B7, B9, B11]
        ensemble = _ensemble_of(self)
        sel = _outputs_of(self)
        if _needs_grad(frames + self._all_tensors()):
            if ensemble is not None:
                raise BinB200Error(f"self-ensemble {ensemble!r} is inference-only: call the net under torch.no_grad(), "
                                   "or set_self_ensemble(net, None) to train")
            if sel is not None:
                raise BinB200Error(f"output selection {sel[0]} is inference-only: call the net under torch.no_grad(), "
                                   "or set_outputs(net, None) to train")
            from .autograd import window_apply
            return window_apply(self, frames)
        frames = [f.contiguous() for f in frames]
        _check_frames(frames)
        wanted = range(14) if sel is None else sel[0]
        live = _window_live(wanted)
        if ensemble is not None:
            outs = self._forward_flipx4(frames, live, wanted)
        elif _graphs_enabled() and not getattr(self, "_is_replica", False) and not torch.cuda.is_current_stream_capturing():
            outs = self._forward_graphed(frames, live, wanted)
        else:
            outs = _window_fwd(self, frames, live)
        return tuple(outs) if sel is None else _selected(outs, sel)

    def _forward_flipx4(self, frames, live, wanted):
        """x4 flip self-ensemble (utils/test_util.py:110-132 flipx4_forward, applied to all 6 frames and the wanted
        outputs): the four orientations run as ONE window at batch 4B, then each output is flipped back and averaged.
        Eager, not graphed: a graph capture would hold a second batch-4B workspace (about 25 GB at 768x1344) in its
        private pool."""
        with torch.cuda.device(frames[0].device):
            big = ops.flipx4_expand(frames)
            outs = _window_fwd(self, big, live)
            del big
            return _flipx4_mean_at(outs, wanted)

    def _forward_graphed(self, frames, live, wanted):
        """The ~340 kernel launches of a window are captured once per (shape, weight version, live nodes) into a
        CUDA graph and replayed: removes ~10 % of host launch overhead at 720p.  Inputs are copied
        into the graph's static buffers, the wanted outputs are returned as fresh tensors (SURVEY 8b)."""
        dev = frames[0].device
        key = (dev.index, tuple(frames[0].shape), _prec_of(self), live,
               tuple((p.data_ptr(), p._version) for p in self._all_tensors()))
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
                    _window_fwd(self, static_in, live)
                    _WS.pop(_ws_key(dev), None)                     # the side stream's scratch buffer is not needed again
                torch.cuda.current_stream().wait_stream(side)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    static_out = _window_fwd(self, static_in, live)
                    ws = _WS.pop(_ws_key(dev), None)                # owned by this entry (graph-private memory pool)
                ent = {"key": key, "graph": graph, "in": static_in, "out": static_out, "ws": ws}
                self.__dict__["_graph_entry"] = ent
            else:
                for d, f in zip(ent["in"], frames):
                    d.copy_(f)
            ent["graph"].replay()
            return [ent["out"][i].clone() if i in wanted else None for i in range(14)]

    def forward_pyramid3(self, B1, B3, B5, B7):
        """BASELINE config 2a: stages 1-3 on 4 frames -> [I2',I4',I6',I3',I5',I4''] (SURVEY 8d)."""
        if _ensemble_of(self) is not None:
            raise BinB200Error("forward_pyramid3 has no self-ensemble mode; set_self_ensemble(net, None) first")
        pyr = self.model
        if _needs_grad([B1, B3, B5, B7] + [p for m in (pyr.model1_1, pyr.model2_1, pyr.model3_1) for p in m._conv_params()]):
            from .autograd import pyramid3_apply                      # BASELINE config 3a (training on the 4-frame graph)
            return pyramid3_apply(self, (B1, B3, B5, B7))
        # every stage in fp16, whatever set_precision says
        return _pyramid3_schedule(lambda m, calls: _batched(m, calls, prec=0), pyr, (B1, B3, B5, B7))


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


UNWANTED = ("none", "zeros")


def _outputs_of(module) -> Optional[Tuple[Tuple[int, ...], str]]:
    """`module.outputs`: None (all 14 outputs) or (the wanted indices in ascending order, "none" | "zeros")."""
    sel = getattr(module, "outputs", None)
    if sel is None:
        return None
    ok = (isinstance(sel, tuple) and len(sel) == 2 and isinstance(sel[0], tuple) and sel[0] and sel[1] in UNWANTED
          and all(type(i) is int and 0 <= i < 14 for i in sel[0]) and list(sel[0]) == sorted(set(sel[0])))
    if not ok:
        raise BinB200Error(f"unknown output selection {sel!r}; set it with set_outputs(net, indices, unwanted)")
    return sel


def _flipx4_mean_at(outs, wanted) -> list:
    """ops.flipx4_mean of the outputs `wanted` of a batch-4B window, at their positions of a 14-list; None elsewhere."""
    means = [None] * 14
    for i, m in zip(wanted, ops.flipx4_mean([outs[i] for i in wanted])):
        means[i] = m
    return means


def _selected(outs, sel) -> tuple:
    """The 14-tuple a net with the selection `sel` returns: outs[i] at the wanted positions; elsewhere None, or with
    unwanted="zeros" one shared all-zero view of an output's shape, backed by a single element."""
    wanted, unwanted = sel
    like = outs[wanted[0]]
    rest = torch.zeros((), device=like.device).expand(like.shape) if unwanted == "zeros" else None
    return tuple(outs[i] if i in wanted else rest for i in range(14))


def set_outputs(net: nn.Module, indices, unwanted: str = "none") -> nn.Module:
    """Compute only the outputs a caller reads, for every window net in `net.modules()` (so a DataParallel wrapper or a
    model object holding the net works).  `indices`: distinct positions 0..13 of the 14-tuple, or None for all 14 (the
    default).  A call still returns a 14-tuple: the wanted positions hold the same bits as without a selection, and the
    backbone calls and ConvLSTM cells that no wanted output depends on do not run (13 of the 17 calls for (13, 8, 12),
    the three images test.py writes).  The other positions hold None (unwanted="none"), so a wrong index fails loudly,
    or one shared all-zero (B,3,H,W) view of a single element (unwanted="zeros"), for test.py and demo.py run unchanged:
    they convert Ft_p[7] and Ft_p[9] to images they never use.  StreamingBIN follows the selection.  Inference only: a
    grad-enabled call then raises.  It is a plain attribute, not a parameter or buffer: the state_dict is unchanged."""
    if unwanted not in UNWANTED:
        raise BinB200Error(f"unknown unwanted mode {unwanted!r}; use 'none' or 'zeros'")
    sel = None
    if indices is not None:
        try:
            idx = list(indices)
        except TypeError:
            raise BinB200Error(f"set_outputs: indices must be an iterable of ints in 0..13 or None; got {indices!r}") from None
        if not idx:
            raise BinB200Error("set_outputs: the selection is empty; pass None for all 14 outputs")
        if any(type(i) is not int or not 0 <= i < 14 for i in idx) or len(set(idx)) != len(idx):
            raise BinB200Error(f"set_outputs: indices must be distinct ints in 0..13; got {indices!r}")
        sel = (tuple(sorted(idx)), unwanted)
    nets = [m for m in net.modules() if isinstance(m, RDN_residual_interp_5_input_ConvLSTM_L)]
    if not nets:
        raise BinB200Error("set_outputs: no RDN_residual_interp_5_input_ConvLSTM_L in this module")
    for m in nets:
        m.outputs = sel
    return net
