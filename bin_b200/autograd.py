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
from .ops import _stream
from .rdn import (_LSTM_NAMES, _check_frames, _checkpointing_of, _launch_stage, _pyramid3_schedule, _pyramid_schedule,
                  _window_schedule)

LOSS_SCALE_TARGET = 2048.0    # max|dOut| * scale after loss scaling (fp16: 32x headroom to 65504; deep-layer gradients stay normal)
_loss_scale_target = LOSS_SCALE_TARGET


def loss_scale_target() -> float:
    """What each backbone backward scales max|dOut| to.  LOSS_SCALE_TARGET unless set_loss_scale_target, or
    bin_b200.optim.Adam(loss_scale_backoff=True) after a skipped step, has lowered it."""
    return _loss_scale_target


def set_loss_scale_target(x: float) -> None:
    """A smaller target leaves more of fp16's range above the scaled gradients and pushes the small ones towards the
    subnormals.  Takes effect at the next backward; 1 <= x <= LOSS_SCALE_TARGET."""
    global _loss_scale_target
    if not 1.0 <= x <= LOSS_SCALE_TARGET:
        raise ValueError(f"loss-scale target must lie in [1, {LOSS_SCALE_TARGET:g}]")
    _loss_scale_target = float(x)


def deterministic_flags() -> int:
    """BIN_DETERMINISTIC when torch.use_deterministic_algorithms(True) is in force, read at the call that reduces: the loss,
    bias and ConvLSTM gradient sums then run in a fixed order and the weight gradients on a grid independent of the SM
    count (DESIGN.md §4f).  0 otherwise: the default atomic sums."""
    return _lib.BIN_DETERMINISTIC if torch.are_deterministic_algorithms_enabled() else 0


def _input_key(model, frames):
    """What a recomputing backward must find unchanged: the weights and the stage's input frames (pointer, version)."""
    return tuple((t.data_ptr(), t._version) for t in list(model._conv_params()) + list(frames))


def grad_plan(needs_input_grad, ncalls: int, nframes: int, nconv: int = _lib.BIN_BACKBONE_NCONV):
    """What one BackboneStageFn backward computes, from its ctx.needs_input_grad = (model, ncalls, *frames, *params):
    (need, frame_needed).  need is the 2 * nconv-byte host mask of bin_backbone_bwd_masked (nconv = the backbone's
    bin_backbone_nconv), 1 where a parameter (weight then bias of each conv, the order of _conv_params) wants its
    gradient; frame_needed[k][f] says whether frame f of call k does (its dframes pointer is NULL when not)."""
    nf = ncalls * nframes
    flags = tuple(needs_input_grad)[2:]
    if len(flags) != nf + 2 * nconv:
        raise BinB200Error(f"grad_plan: expected {nf + 2 * nconv} inputs after (model, ncalls), got {len(flags)}")
    frame_needed = [[bool(flags[k * nframes + f]) for f in range(nframes)] for k in range(ncalls)]
    need = (C.c_ubyte * (2 * nconv))(*[1 if x else 0 for x in flags[nf:]])
    return need, frame_needed


def _grad_frames(dframes, B: int) -> _lib.Frames:
    """dframes table of a backward: None entries become NULL pointers (no gradient for that frame)."""
    fr = _lib.Frames()
    fr.ncalls, fr.nframes, fr.Bc = len(dframes), len(dframes[0]), B
    for k, call in enumerate(dframes):
        for f, t in enumerate(call):
            fr.frame[k][f] = None if t is None else t.data_ptr()
    return fr


class BackboneStageFn(torch.autograd.Function):
    """ncalls same-weight backbone calls (RDN.py:210-334) in one launch, with backward.

    Default: the forward keeps the stage's whole training workspace (all its RDBs' growth maps) until the backward.
    With set_activation_checkpointing(net, "recompute") it keeps only its input frames: the forward is the inference
    forward into the shared per-stream workspace, and the backward runs that forward again and rebuilds each RDB's
    growth maps just before that RDB's backward.  Every kernel sees the same operands in both (DESIGN.md §4e).

    Frozen tensors (requires_grad False) get no gradient and cost no work: the backward computes only what
    ctx.needs_input_grad asks for (DESIGN.md §4g).  A stage none of whose inputs needs a gradient runs the inference
    forward, with the fused RDB tail, and keeps nothing for a backward."""

    @staticmethod
    def forward(ctx, model, ncalls: int, *args):
        n, arch = model.NFRAMES, model.arch
        frames = [a.detach().contiguous() for a in args[: ncalls * n]]
        calls = [frames[k * n:(k + 1) * n] for k in range(ncalls)]
        B, _, H, W = frames[0].shape
        dev = frames[0].device
        # training runs in fp16 whatever set_precision says: the backward kernels have no fp32 (x3) mode
        if not any(ctx.needs_input_grad[2:]):
            with torch.cuda.device(dev):
                outs = [torch.empty_like(frames[0]) for _ in range(ncalls)]
                _launch_stage(model, calls, outs, prec=0)
            return tuple(outs)
        recompute = _checkpointing_of(model) == "recompute"
        with torch.cuda.device(dev):
            outs = [torch.empty_like(frames[0]) for _ in range(ncalls)]
            if recompute:
                _launch_stage(model, calls, outs, prec=0)
                save = None
            else:
                fr = ops.make_frames(calls, outs)
                nbytes = lib().bin_backbone_train_workspace_bytes(arch, B * ncalls, H, W)
                save = torch.empty(nbytes, dtype=torch.uint8, device=dev)          # owned by this node until backward
                check(lib().bin_backbone_fwd_train(arch, model.packed_blob().data_ptr(), C.byref(fr), H, W, save.data_ptr(),
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
        n, arch = model.NFRAMES, model.arch
        dev = ctx.dev
        flags = deterministic_flags()
        with torch.cuda.device(dev):
            gouts = [torch.zeros((B, 3, H, W), device=dev) if g is None else g.contiguous().float() for g in gouts]
            # bin_grad_scale reads float4s: a contiguous view at an offset (e.g. a slice of a flat buffer) gets a copy
            gouts = [g if g.data_ptr() % 16 == 0 else g.clone() for g in gouts]
            sbuf = torch.empty(2, device=dev)                                    # [scale, scratch]; stays on the device
            gp = (C.c_void_p * ncalls)(*[g.data_ptr() for g in gouts])
            check(lib().bin_grad_scale(gp, ncalls, gouts[0].numel(), loss_scale_target(), sbuf.data_ptr(),
                                       sbuf.data_ptr() + 4, _stream()))
            scale = sbuf[:1]
            need, frame_needed = grad_plan(ctx.needs_input_grad, ncalls, n, model.nconv)
            dframes = [[torch.empty((B, 3, H, W), device=dev) if want else None for want in call] for call in frame_needed]
            dout = ops.make_frames([[g] * n for g in gouts], gouts)             # only .out / ncalls / Bc are read
            dfr = _grad_frames(dframes, B)
            gparams = torch.zeros(lib().bin_backbone_grad_param_floats(arch), device=dev) if any(need) else None
            gp_ptr = None if gparams is None else gparams.data_ptr()
            gws = torch.empty(lib().bin_backbone_grad_workspace_bytes(arch, B * ncalls, H, W), dtype=torch.uint8, device=dev)
            if recompute:
                frames = ctx.frames_keepalive
                calls = [frames[k * n:(k + 1) * n] for k in range(ncalls)]
                scratch = [torch.empty_like(frames[0]) for _ in range(ncalls)]   # the forward's outputs stay untouched
                ws = _launch_stage(model, calls, scratch, prec=0)                  # fp16, as in the forward
                check(lib().bin_backbone_bwd_recompute_masked(arch, model.packed_blob().data_ptr(),
                                                              model._cached_pack("t").data_ptr(), C.byref(dout),
                                                              C.byref(dfr), H, W, ws.data_ptr(), ws.numel(),
                                                              gws.data_ptr(), gws.numel(), gp_ptr, scale.data_ptr(),
                                                              flags, need, _stream()))
            else:
                check(lib().bin_backbone_bwd_masked(arch, model._cached_pack("t").data_ptr(), C.byref(dout), C.byref(dfr), H, W,
                                                    ctx.save.data_ptr(), gws.data_ptr(), gws.numel(), gp_ptr,
                                                    scale.data_ptr(), flags, need, _stream()))
        ctx.save = None
        pgrads, off = [], 0
        for p, want in zip(model._conv_params(), need):
            pgrads.append(gparams[off:off + p.numel()].view_as(p) if want else None)
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
            # a gradient nobody asked for is a NULL output: the library skips the pass that only it needs
            need_x, need_w, need_b, need_cp, need_hp = ctx.needs_input_grad
            dgates = torch.empty((B, 12, H, W), device=dev)
            dx = torch.empty_like(x) if need_x else None
            dcp = torch.empty_like(x) if ctx.has_state and need_cp else None
            dhp = torch.empty_like(x) if ctx.has_state and need_hp else None
            dw = torch.zeros_like(w) if need_w else None
            db = torch.zeros_like(b) if need_b else None
            flags = deterministic_flags()
            scratch = (torch.empty(lib().bin_convlstm_bwd_scratch_bytes(B, H, W), dtype=torch.uint8, device=dev)
                       if flags and (need_w or need_b) else None)
            P = lambda t: None if t is None else t.data_ptr()
            check(lib().bin_convlstm_bwd_ex(x.data_ptr(), P(cp), P(hp), w.data_ptr(), b.data_ptr(), P(dh), P(dc),
                                            dgates.data_ptr(), P(dx), P(dcp), P(dhp), P(dw), P(db),
                                            B, H, W, flags, P(scratch), 0 if scratch is None else scratch.numel(),
                                            _stream()))
        return dx, dw, db, dcp, dhp


def convlstm_apply(module, x, state):
    cp, hp = (None, None) if state is None else (state[0], state[1])
    h, c = ConvLSTMFn.apply(x, module.Gates.weight, module.Gates.bias, cp, hp)
    return h, [c, h]


def pyramid_apply(pyr, B1, B3, B5, B7, B9, previous_input=None):
    """RDN_residual_interp_5_input.forward (RDN.py:367-405) with autograd, 4 batched stage launches."""
    return _pyramid_schedule(backbone_stage, pyr, B1, B3, B5, B7, B9, previous_input)


def pyramid3_apply(module, F):
    """Stages 1-3 on 4 frames with autograd (BASELINE config 2a/3a; pattern of RDN.py:383-387)."""
    return _pyramid3_schedule(backbone_stage, module.model, F)


def window_apply(module, F):
    """Grad-enabled RDN_residual_interp_5_input_ConvLSTM_L.forward (RDN.py:422-465): the same 17 unique
    backbone calls / 6 live ConvLSTM calls as the inference window (SURVEY App. A), each batched stage an autograd node
    and each ConvLSTM cell its own."""
    F = [f.contiguous() for f in F]
    _check_frames(F)
    pyr = module.model
    cells = [getattr(module, n) for n in _LSTM_NAMES]
    s1 = backbone_stage(pyr.model1_1, [(F[0], F[1]), (F[1], F[2]), (F[2], F[3]), (F[3], F[4]), (F[4], F[5])])
    lstm = lambda group: [convlstm_apply(cells[k], x, None)[0] for k, x in group]
    return _window_schedule(backbone_stage, lstm, pyr, F, s1)
