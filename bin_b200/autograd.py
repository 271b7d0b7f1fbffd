"""torch.autograd.Functions of the BIN hot path (training step, BASELINE config 3).

Each batched backbone launch (same-weight calls riding along N) is one autograd node; PyTorch's
autograd engine only routes the 14 outputs' gradients through the temporal DAG (summing frames that
feed several calls).  All arithmetic -- forward, data gradients, weight gradients -- runs in
libbin_b200.so; nothing here falls back to PyTorch ops for the math.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Sequence

import torch

from . import _lib, ops
from ._lib import BinB200Error, check, lib

LOSS_SCALE_TARGET = 2048.0    # max|dOut| * scale after loss scaling (fp16: 32x headroom to 65504; deep-layer gradients stay normal)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def deterministic_flags() -> int:
    """BIN_DETERMINISTIC when torch.use_deterministic_algorithms(True) is in force, read at the call that reduces: the loss,
    bias and ConvLSTM gradient sums then run in a fixed order and the weight gradients on a grid independent of the SM
    count (DESIGN.md §4f).  0 otherwise: the default atomic sums."""
    return _lib.BIN_DETERMINISTIC if torch.are_deterministic_algorithms_enabled() else 0


def _packed_t(model) -> torch.Tensor:
    ps = model._conv_params()
    key = (ps[0].device.index,) + tuple((p.data_ptr(), p._version) for p in ps)
    cached = model.__dict__.get("_packed_t")
    if cached is None or cached[0] != key:
        dev = ps[0].device
        blob = torch.empty(lib().bin_backbone_packed_t_bytes(model.NFRAMES), dtype=torch.uint8, device=dev)
        wp = (C.c_void_p * _lib.BIN_BACKBONE_NCONV)(*[p.data_ptr() for p in ps[0::2]])
        check(lib().bin_backbone_pack_t(model.NFRAMES, wp, blob.data_ptr(), _stream()))
        model.__dict__["_packed_t"] = (key, blob)
        cached = model.__dict__["_packed_t"]
    return cached[1]


def _input_key(model, frames):
    """What a recomputing backward must find unchanged: the weights and the stage's input frames (pointer, version)."""
    return tuple((t.data_ptr(), t._version) for t in list(model._conv_params()) + list(frames))


def _inference_fwd(model, calls, outs, B, H, W, dev) -> torch.Tensor:
    """bin_backbone_fwd of one batched stage into the shared per-(device, stream) workspace, which it returns."""
    from .rdn import _workspace
    n = model.NFRAMES
    fr = ops.make_frames(calls, outs)
    ws = _workspace(dev, lib().bin_backbone_workspace_bytes(n, B * len(calls), H, W))
    check(lib().bin_backbone_fwd(n, model.packed_blob().data_ptr(), C.byref(fr), H, W, ws.data_ptr(), ws.numel(),
                                 _stream()))
    return ws


class BackboneStageFn(torch.autograd.Function):
    """ncalls same-weight backbone calls (RDN.py:210-334) in one launch, with backward.

    Default: the forward keeps the stage's whole training workspace (all 12 RDBs' growth maps) until the backward.
    With set_activation_checkpointing(net, "recompute") it keeps only its input frames: the forward is the inference
    forward into the shared per-stream workspace, and the backward runs that forward again and rebuilds each RDB's
    growth maps just before that RDB's backward.  Every kernel sees the same operands in both (DESIGN.md §4e)."""

    @staticmethod
    def forward(ctx, model, ncalls: int, *args):
        from .rdn import _checkpointing_of
        n = model.NFRAMES
        frames = [a.detach().contiguous() for a in args[: ncalls * n]]
        calls = [frames[k * n:(k + 1) * n] for k in range(ncalls)]
        B, _, H, W = frames[0].shape
        dev = frames[0].device
        recompute = _checkpointing_of(model) == "recompute"
        with torch.cuda.device(dev):
            outs = [torch.empty_like(frames[0]) for _ in range(ncalls)]
            if recompute:
                _inference_fwd(model, calls, outs, B, H, W, dev)
                save = None
            else:
                fr = ops.make_frames(calls, outs)
                nbytes = lib().bin_backbone_train_workspace_bytes(n, B * ncalls, H, W)
                save = torch.empty(nbytes, dtype=torch.uint8, device=dev)          # owned by this node until backward
                check(lib().bin_backbone_fwd_train(n, model.packed_blob().data_ptr(), C.byref(fr), H, W, save.data_ptr(),
                                                   save.numel(), _stream()))
        ctx.model, ctx.ncalls, ctx.save, ctx.shape, ctx.dev = model, ncalls, save, (B, H, W), dev
        ctx.recompute_key = _input_key(model, frames) if recompute else None
        ctx.frames_keepalive = frames
        return tuple(outs)

    @staticmethod
    def backward(ctx, *gouts):
        model, ncalls, (B, H, W) = ctx.model, ctx.ncalls, ctx.shape
        recompute = ctx.recompute_key is not None
        if recompute:
            # every input of the recomputation is still held (frames_keepalive, the weights), so a second backward
            # (retain_graph) recomputes the same activations and gives the same gradients
            if _input_key(model, ctx.frames_keepalive) != ctx.recompute_key:
                raise BinB200Error("bin_b200: a backbone weight or input frame was modified in place between the forward "
                                   "and the backward; activation recomputation would give wrong gradients")
        elif ctx.save is None:
            raise BinB200Error("bin_b200: backward through a backbone stage twice (retain_graph / double backward) is not "
                               "supported: the saved activations are released after the first backward")
        n = model.NFRAMES
        dev = ctx.dev
        flags = deterministic_flags()
        with torch.cuda.device(dev):
            gouts = [torch.zeros((B, 3, H, W), device=dev) if g is None else g.contiguous().float() for g in gouts]
            sbuf = torch.empty(2, device=dev)                                    # [scale, scratch]; stays on the device
            gp = (C.c_void_p * ncalls)(*[g.data_ptr() for g in gouts])
            check(lib().bin_grad_scale(gp, ncalls, gouts[0].numel(), LOSS_SCALE_TARGET, sbuf.data_ptr(),
                                       sbuf.data_ptr() + 4, _stream()))
            scale = sbuf[:1]
            dframes = [[torch.empty((B, 3, H, W), device=dev) for _ in range(n)] for _ in range(ncalls)]
            dout = ops.make_frames([[g] * n for g in gouts], gouts)             # only .out / ncalls / Bc are read
            dfr = ops.make_frames(dframes, [None] * ncalls)
            gparams = torch.zeros(lib().bin_backbone_grad_param_floats(n), device=dev)
            gws = torch.empty(lib().bin_backbone_grad_workspace_bytes(n, B * ncalls, H, W), dtype=torch.uint8, device=dev)
            if recompute:
                frames = ctx.frames_keepalive
                calls = [frames[k * n:(k + 1) * n] for k in range(ncalls)]
                scratch = [torch.empty_like(frames[0]) for _ in range(ncalls)]   # the forward's outputs stay untouched
                ws = _inference_fwd(model, calls, scratch, B, H, W, dev)
                check(lib().bin_backbone_bwd_recompute_ex(n, model.packed_blob().data_ptr(), _packed_t(model).data_ptr(),
                                                          C.byref(dout), C.byref(dfr), H, W, ws.data_ptr(), ws.numel(),
                                                          gws.data_ptr(), gws.numel(), gparams.data_ptr(), scale.data_ptr(),
                                                          flags, _stream()))
            else:
                check(lib().bin_backbone_bwd_ex(n, _packed_t(model).data_ptr(), C.byref(dout), C.byref(dfr), H, W,
                                                ctx.save.data_ptr(), gws.data_ptr(), gws.numel(), gparams.data_ptr(),
                                                scale.data_ptr(), flags, _stream()))
        ctx.save = None
        pgrads, off = [], 0
        for p in model._conv_params():
            pgrads.append(gparams[off:off + p.numel()].view_as(p))
            off += p.numel()
        flat = [g for call in dframes for g in call]
        return (None, None, *flat, *pgrads)


def backbone_stage(model, calls: Sequence[Sequence[torch.Tensor]]) -> List[torch.Tensor]:
    flat = [t for c in calls for t in c]
    # the weights are passed as the module's ATTRIBUTES (replica-safe, see _Backbone._conv_params): in an nn.DataParallel
    # replica they are Broadcast outputs whose gradients autograd reduces onto the master parameters
    return list(BackboneStageFn.apply(model, len(calls), *flat, *model._conv_params()))


def backbone_apply(module, frames):
    return backbone_stage(module, [list(frames)])[0]


class ConvLSTMFn(torch.autograd.Function):
    """ConvLSTMCell.forward (RDN.py:50-95) with backward; returns (h', c')."""

    @staticmethod
    def forward(ctx, x, w, b, c_prev, h_prev):
        x = x.detach().contiguous()
        state = None if c_prev is None else (c_prev.detach().contiguous(), h_prev.detach().contiguous())
        h, c = ops.convlstm_fwd(x, w.detach(), b.detach(), state)
        ctx.save_for_backward(x, w.detach(), b.detach(), *(state if state is not None else ()))
        ctx.has_state = state is not None
        return h, c

    @staticmethod
    def backward(ctx, dh, dc):
        saved = ctx.saved_tensors
        x, w, b = saved[0], saved[1], saved[2]
        cp, hp = (saved[3], saved[4]) if ctx.has_state else (None, None)
        B, _, H, W = x.shape
        dev = x.device
        with torch.cuda.device(dev):
            dh = None if dh is None else dh.contiguous().float()
            dc = None if dc is None else dc.contiguous().float()
            dgates = torch.empty((B, 12, H, W), device=dev)
            dx = torch.empty_like(x)
            dcp = torch.empty_like(x) if ctx.has_state else None
            dhp = torch.empty_like(x) if ctx.has_state else None
            dw = torch.zeros_like(w)
            db = torch.zeros_like(b)
            flags = deterministic_flags()
            scratch = (torch.empty(lib().bin_convlstm_bwd_scratch_bytes(B, H, W), dtype=torch.uint8, device=dev)
                       if flags else None)
            P = lambda t: None if t is None else t.data_ptr()
            check(lib().bin_convlstm_bwd_ex(x.data_ptr(), P(cp), P(hp), w.data_ptr(), b.data_ptr(), P(dh), P(dc),
                                            dgates.data_ptr(), dx.data_ptr(), P(dcp), P(dhp), dw.data_ptr(), db.data_ptr(),
                                            B, H, W, flags, P(scratch), 0 if scratch is None else scratch.numel(),
                                            _stream()))
        return dx, dw, db, dcp, dhp


def convlstm_apply(module, x, state):
    cp, hp = (None, None) if state is None else (state[0], state[1])
    h, c = ConvLSTMFn.apply(x, module.Gates.weight, module.Gates.bias, cp, hp)
    return h, [c, h]


def pyramid_apply(pyr, B1, B3, B5, B7, B9, previous_input=None):
    """RDN_residual_interp_5_input.forward (RDN.py:367-405) with autograd, 4 batched stage launches."""
    m1, m2, m3, m4 = pyr.model1_1, pyr.model2_1, pyr.model3_1, pyr.model4_1
    I2, I4, I6, I8 = backbone_stage(m1, [(B1, B3), (B3, B5), (B5, B7), (B7, B9)])
    if previous_input is not None and previous_input[0] is not None:
        p4, p6, p8, p5, p7, p6b = previous_input
        I3, I5, I7 = backbone_stage(m2, [(p4, I2, I4), (p6, I4, I6), (p8, I6, I8)])
        I4b, I6b = backbone_stage(m3, [(p5, B3, I3, I5, B5), (p7, B5, I5, I7, B7)])
        (I5c,) = backbone_stage(m4, [(p6b, I4, I4b, I6b, I6)])
    else:
        I3, I5, I7 = backbone_stage(m2, [(I2, I2, I4), (I4, I4, I6), (I6, I6, I8)])
        I4b, I6b = backbone_stage(m3, [(I3, B3, I3, I5, B5), (I5, B5, I5, I7, B7)])
        (I5c,) = backbone_stage(m4, [(I4, I4, I4b, I6b, I6)])
    return I2, I4, I6, I8, I3, I5, I7, I4b, I6b, I5c


def pyramid3_apply(module, F):
    """Stages 1-3 on 4 frames with autograd (BASELINE config 2a/3a; pattern of RDN.py:383-387)."""
    pyr = module.model
    o0, o1, o2 = backbone_stage(pyr.model1_1, [(F[0], F[1]), (F[1], F[2]), (F[2], F[3])])
    o3, o4 = backbone_stage(pyr.model2_1, [(o0, o0, o1), (o1, o1, o2)])
    (o5,) = backbone_stage(pyr.model3_1, [(o3, F[1], o3, o4, F[2])])
    return o0, o1, o2, o3, o4, o5


def window_apply(module, F):
    """Grad-enabled RDN_residual_interp_5_input_ConvLSTM_L.forward (RDN.py:422-465): the same 17 unique
    backbone calls / 6 live ConvLSTM calls as bin_window_fwd (SURVEY App. A), each batched stage an autograd node."""
    from .rdn import _LSTM_NAMES, _check_frames
    F = [f.contiguous() for f in F]
    _check_frames(F)
    pyr = module.model
    m1, m2, m3, m4 = pyr.model1_1, pyr.model2_1, pyr.model3_1, pyr.model4_1
    cells = [getattr(module, n) for n in _LSTM_NAMES]
    lstm = lambda k, x: convlstm_apply(cells[k], x, None)[0]
    o = [None] * 14
    o[0], o[1], o[2], o[3], o[10] = backbone_stage(m1, [(F[0], F[1]), (F[1], F[2]), (F[2], F[3]), (F[3], F[4]), (F[4], F[5])])
    p4, p6, p8 = lstm(0, o[1]), lstm(1, o[2]), lstm(2, o[3])
    o[4], o[5], o[6], t0, t1, o[11] = backbone_stage(m2, [(o[0], o[0], o[1]), (o[1], o[1], o[2]), (o[2], o[2], o[3]),
                                                          (p4, o[1], o[2]), (p6, o[2], o[3]), (p8, o[3], o[10])])
    p5, p7 = lstm(3, o[5]), lstm(4, o[6])
    o[7], o[8], t2, o[12] = backbone_stage(m3, [(o[4], F[1], o[4], o[5], F[2]), (o[5], F[2], o[5], o[6], F[3]),
                                              (p5, F[2], t0, t1, F[3]), (p7, F[3], t1, o[11], F[4])])
    p6b = lstm(5, o[8])
    o[9], o[13] = backbone_stage(m4, [(o[1], o[1], o[7], o[8], o[2]), (p6b, o[2], t2, o[12], o[3])])
    return tuple(o)
