"""TEST INFRASTRUCTURE: backbone weights with no ReLU input near 0, their fp64 gradients, and the per-tensor gradient bar.

fp16 storage moves every RDB growth-conv pre-activation by a rounding error; where one sits near 0 the CUDA path and
the fp64 oracle can take different sides of the ReLU, and no per-tensor bar survives that.  no_flip_sd rebuilds the
growth convs of a synthetic backbone (any width G0 and depth D, oracle/arch_oracle.py) so that, on the given calls,
every ReLU input is at least DELTA away from 0; check_no_relu_near_zero asserts it on the fp32 weights the backbone
runs.  oracle_grads is fp64 autograd through arch_oracle.backbone, optionally with the fp16-storage emulation of
bin_oracle (activations and loss-scaled gradients rounded to fp16 where the CUDA path stores them).

no_flip_window_sd does the same for a whole six-frame window: each of the four canonical backbones is rebuilt on the
calls the window makes of it, in dataflow order, so that later stages are built on what earlier ones give.
window_oracle_grads is fp64 autograd through that window, either along the reference's own dataflow or along the
library's batched schedule (bin_b200.rdn._window_schedule), where the fp16-storage emulation rounds the gradients of all
the calls of a stage at one scale, as the library does.

check_gradients holds a set of gradients to the bar of the whole-backbone tests: per tensor,
e <= k_emu * e_emu + 1e-3 * max|ref|, with e the CUDA error against fp64, e_emu the emulating oracle's and k_emu = 4
for the bias of growth convs 0-2 (whose dY is summed in fp16, in place, over several launches, where the oracle rounds
the finished sum once) and 2 otherwise.  The bar is normalised by the tensor's max, so a wrong last row or column of a
frame gradient could hide under it; the frame gradients' border bands are held to the same formula, each band with
its own max|ref| and its own e_emu.
"""
from __future__ import annotations

import contextlib
import math

import torch
import torch.nn.functional as F

from oracle import arch_oracle as A
from oracle import bin_oracle as O

BETA = 0.05              # |bias| of every growth conv channel
TARGET = 0.1 * BETA      # the construction puts the smallest "on" pre-activation here
DELTA = 0.05 * BETA      # margin asserted on every run: every ReLU input is >= DELTA or <= -DELTA
MIN_CV = 0.2             # every "on" channel: spatial std >= 20 % of its mean, where it has more than one pixel per item
TILE_ROWS = 8            # output rows of a conv tile (internal.h)
TILE_COLS_5X5 = 28       # output columns of a 5x5 conv tile: SFENet1's data gradient writes the packed frame gradient


def rdb_input(frames, sd):
    return O.conv(O.conv(O.space_to_depth2(torch.cat(list(frames), 1)), sd, "SFENet1"), sd, "SFENet2")


def no_flip_sd(n, seed, calls, g0=O.G0, d=O.D):
    """A.synth_backbone_sd(n, seed, g0, d) with the 4 d RDB growth convs rebuilt, in fp64 on these calls' frames, so
    that no ReLU input is near 0: each channel's 3x3 taps lose their mean (a locally constant input then gives ~0, which
    centres the channel), half the channels ("on", the 16 whose pre-activations have the lightest tail, flipped to point
    down) get bias +BETA and a scale that puts their smallest pre-activation at TARGET (if all of a channel's
    pre-activations lie on one side of the bias, the one farthest from it), the rest bias -BETA and a scale
    that keeps them within [-1.5 BETA, -0.5 BETA].  The statistics of a channel are pooled over every call, batch item
    and pixel.  Returns fp32 weights on the calls' device."""
    dev = calls[0][0].device
    sd = {k: v.to(dev, torch.float64) for k, v in A.synth_backbone_sd(n, seed, g0, d).items()}
    xs = [rdb_input(c, sd) for c in calls]
    for i in range(d):
        feats = xs
        for c in range(O.C):
            name = f"RDBs.{i}.convs.{c}.conv.0"
            w = sd[name + ".weight"]
            w = w - w.mean((2, 3), keepdim=True)
            u = torch.cat([F.conv2d(f, w, padding=1).transpose(0, 1).flatten(1) for f in feats], 1)
            mu, sig, umin, umax = u.mean(1), u.std(1), u.min(1).values, u.max(1).values
            sign = torch.where(mu - umin <= umax - mu, 1.0, -1.0).to(u)
            tail = torch.minimum(mu - umin, umax - mu) / sig
            on = torch.zeros(O.G, dtype=torch.bool, device=dev)
            on[tail.argsort()[:O.G // 2]] = True
            lowest = torch.where(sign > 0, umin, -umax)
            # a channel whose u never crosses 0 (a map of one row or column, where most taps read the zero padding)
            # has no tail below the bias: it is turned round, so that its largest |u| lands at TARGET
            reach = torch.where(lowest < 0, -lowest, -u.abs().max(1).values)
            alpha = torch.where(on, sign * (BETA - TARGET) / reach, 0.5 * BETA / u.abs().max(1).values)
            sd[name + ".weight"] = w * alpha.view(-1, 1, 1, 1)
            sd[name + ".bias"] = torch.where(on, BETA, -BETA).to(u)
            feats = [torch.cat((f, O.conv(f, sd, name).relu()), 1) for f in feats]
        xs = [O.conv(f, sd, f"RDBs.{i}.LFF") + x for f, x in zip(feats, xs)]
    return {k: v.float() for k, v in sd.items()}


def check_no_relu_near_zero(calls, sd, min_cv=MIN_CV):
    """The premise of the per-tensor bar, on the weights as the backbone runs them (fp32 values, fp64 arithmetic): every
    growth-conv pre-activation of every call is >= DELTA ("on" channels, bias > 0) or <= -DELTA, and, where a channel
    has more than one pixel per batch item and min_cv is not None, every "on" channel varies across pixels (std >=
    min_cv of its mean), so tap and pixel shifts in the backward stay visible.  Returns (worst margin, worst std/mean;
    inf where not measured)."""
    dev = calls[0][0].device
    sd = {k: v.to(dev, torch.float64) for k, v in sd.items()}
    feats_x = [rdb_input([f.double() for f in c], sd) for c in calls]
    spatial = feats_x[0].shape[2] * feats_x[0].shape[3] > 1
    worst_margin, worst_cv = math.inf, math.inf
    for i in range(A.backbone_depth(sd)):
        feats = feats_x
        for c in range(O.C):
            name = f"RDBs.{i}.convs.{c}.conv.0"
            on = sd[name + ".bias"] > 0
            z = torch.cat([O.conv(f, sd, name).transpose(0, 1).flatten(1) for f in feats], 1)
            margin = min(z[on].min().item(), -z[~on].max().item())
            assert 12 <= int(on.sum()) <= 20 and margin >= DELTA, (name, int(on.sum()), margin)
            worst_margin = min(worst_margin, margin)
            if spatial and min_cv is not None:
                cv = (z[on].std(1) / z[on].mean(1)).min().item()
                assert cv >= min_cv, (name, cv)
                worst_cv = min(worst_cv, cv)
            feats = [torch.cat((f, O.conv(f, sd, name).relu()), 1) for f in feats]
        feats_x = [O.conv(f, sd, f"RDBs.{i}.LFF") + x for f, x in zip(feats, feats_x)]
    return worst_margin, worst_cv


def oracle_grads(pool, calls_idx, cots, sd, emulate, device="cuda"):
    """fp64 autograd through A.backbone on `device` (optionally with fp16-rounded storage of activations and gradients):
    (outputs, gradient of every pool frame, {parameter name: gradient}).  A cotangent of None leaves that call's output
    out of the loss; a frame that reaches the loss through no call gets a zero gradient."""
    leaves = {k: v.to(device, torch.float64).requires_grad_(True) for k, v in sd.items()}
    fr = [p.to(device, torch.float64).requires_grad_(True) for p in pool]
    with O.emulate_fp16_storage(grads=True) if emulate else contextlib.nullcontext():
        outs = [A.backbone([fr[j] for j in idx], leaves) for idx in calls_idx]
    loss = sum((o * c.to(device, torch.float64)).sum() for o, c in zip(outs, cots) if c is not None)
    names = list(leaves)
    grads = torch.autograd.grad(loss, fr + [leaves[k] for k in names], allow_unused=True)
    grads = [torch.zeros_like(t) if g is None else g for g, t in zip(grads, fr + [leaves[k] for k in names])]
    return [o.detach() for o in outs], list(grads[:len(fr)]), dict(zip(names, grads[len(fr):]))


CANON = tuple(O.BACKBONE_ALIASES)        # the window's four distinct backbones, model1_1 .. model4_1, in stage order


def _window_run(F, stage, lstm):
    """The window's 17 backbone calls and 6 ConvLSTM cells on the six frames F, in the library's schedule: the 5 frame
    pairs as stage 1, then bin_b200.rdn._window_schedule.  stage(name, calls) runs the calls of the backbone `name`
    (one of CANON) and returns their outputs; lstm(group) runs the cells (k, x) of a hand-off and returns their h."""
    from types import SimpleNamespace

    from bin_b200 import rdn
    s1 = stage("model1_1", [(F[a], F[a + 1]) for a in range(5)])
    return list(rdn._window_schedule(stage, lstm, SimpleNamespace(**{m: m for m in CANON}), F, s1))


def no_flip_window_sd(seed, g0, d, frames):
    """A window state_dict (net.model = RDN_residual_interp_5_input(lstm=True, GO=g0, D=d)) whose every backbone has no
    ReLU input near 0 on the calls the window makes of it: the ConvLSTM gates of A.synth_state_dict(seed, g0, d), and
    each canonical backbone rebuilt by no_flip_sd on its calls (duplicates removed: the 5 / 6 / 4 / 2 calls of the
    library's schedule), in dataflow order and fp64, each stage's inputs computed with the fp32 weights of the stages
    before it.  Aliases (O.BACKBONE_ALIASES) share the tensors.  frames: the six frames; fp32 weights on the CPU."""
    dev = frames[0].device
    sd = {k: v for k, v in A.synth_state_dict(seed, g0, d).items() if not k.startswith("model.")}
    cells = {k: v.to(dev, torch.float64) for k, v in sd.items()}
    built = {}

    def stage(name, calls):
        calls = [[f.to(dev, torch.float64) for f in c] for c in calls]
        bsd = no_flip_sd(O.BACKBONE_NFRAMES[name], seed * 1000 + 100 + CANON.index(name), calls, g0, d)
        check_no_relu_near_zero(calls, bsd)
        built[name] = bsd
        bsd = {k: v.double() for k, v in bsd.items()}
        return [A.backbone(c, bsd) for c in calls]

    _window_run([f.to(dev, torch.float64) for f in frames], stage,
                lambda group: [O.convlstm(x, cells, O.LSTM_NAMES[k])[0] for k, x in group])
    for canon, aliases in O.BACKBONE_ALIASES.items():
        bsd = {k: v.cpu() for k, v in built[canon].items()}
        for a in aliases:
            sd.update({f"model.{a}.{k}": v for k, v in bsd.items()})
    return sd


@contextlib.contextmanager
def _no_fp16_emulation():
    prev = O._EMULATE_FP16, O._EMULATE_FP16_GRADS
    O._EMULATE_FP16 = O._EMULATE_FP16_GRADS = False
    try:
        yield
    finally:
        O._EMULATE_FP16, O._EMULATE_FP16_GRADS = prev


def window_oracle_grads(frames, cots, sd, emulate, device="cuda", batched=None, wrap=None):
    """fp64 autograd through the six-frame window on `device` (optionally with the fp16-storage emulation of activations
    and gradients): (the 14 outputs, the 6 frame gradients, {parameter name: gradient}), one gradient for each distinct
    tensor of sd under its first name, the names of net.named_parameters(): aliases share one leaf.

    cots: the 14 cotangents (None leaves an output out of the loss), or a function of the 14 outputs that returns the
    loss.  batched (default: emulate) chooses the dataflow.  False: A.window_forward, the reference's own 20 backbone
    calls, independent of the code under test.  True: the library's schedule (_window_run), each stage's calls
    concatenated along the batch and run as one A.backbone, so that the emulation's _round_grad_fp16 sees one tensor per
    stage and rounds every call at the loudest call's scale, as bin_grad_scale does; the ConvLSTM cells run without fp16
    rounding of their weights, like the library's fp32 cell.  wrap(stage, lstm, F) -> (stage, lstm) replaces the batched
    schedule's stage and cell functions, F being the six frame leaves (a test injects window-glue faults with it)."""
    batched = emulate if batched is None else batched
    uniq, full = {}, {}
    for k, v in sd.items():
        if v.data_ptr() not in uniq:
            uniq[v.data_ptr()] = (k, v.to(device, torch.float64).requires_grad_(True))
        full[k] = uniq[v.data_ptr()][1]
    fr = [f.to(device, torch.float64).requires_grad_(True) for f in frames]

    def stage(name, calls):
        B = calls[0][0].shape[0]
        slots = [torch.cat([c[j] for c in calls]) for j in range(len(calls[0]))]
        return list(A.backbone(slots, O.sub_sd(full, f"model.{name}")).split(B))

    def lstm(group):
        with _no_fp16_emulation():
            return [O.convlstm(x, full, O.LSTM_NAMES[k])[0] for k, x in group]

    if wrap is not None:
        stage, lstm = wrap(stage, lstm, fr)
    with O.emulate_fp16_storage(grads=True) if emulate else contextlib.nullcontext():
        outs = _window_run(fr, stage, lstm) if batched else A.window_forward(fr, full)
    loss = cots(outs) if callable(cots) else sum((o * c.to(device, torch.float64)).sum()
                                                 for o, c in zip(outs, cots) if c is not None)
    names, leaves = zip(*uniq.values())
    grads = torch.autograd.grad(loss, fr + list(leaves), allow_unused=True)
    grads = [torch.zeros_like(t) if g is None else g for g, t in zip(grads, fr + list(leaves))]
    return [o.detach() for o in outs], grads[:len(fr)], dict(zip(names, grads[len(fr):]))


def k_emu(key):
    return 4.0 if key.endswith("bias") and ".convs." in key and ".convs.3." not in key else 2.0


def frame_bands(H, W):
    """{name: index} of the border bands of a full-resolution (B, 3, H, W) frame gradient: its last row and column, and
    the rows and columns of the last conv tile of SFENet1's data gradient (TILE_ROWS x TILE_COLS_5X5 at half
    resolution; partial unless h or w is a multiple of the tile)."""
    h, w = H // 2, W // 2
    r0, c0 = 2 * (TILE_ROWS * ((h - 1) // TILE_ROWS)), 2 * (TILE_COLS_5X5 * ((w - 1) // TILE_COLS_5X5))
    return {"last row": (Ellipsis, slice(H - 1, H), slice(None)), "last col": (Ellipsis, slice(W - 1, W)),
            "last tile rows": (Ellipsis, slice(r0, H), slice(None)), "last tile cols": (Ellipsis, slice(c0, W))}


def check_gradients(got, ref, emu, frame_max=None):
    """got, ref, emu: {key: gradient}; keys starting with "frame" are (B, 3, H, W) frame gradients and get the border
    bands too.  frame_max: the max|ref| that normalises every frame gradient's 1e-3 term (default: each tensor's or
    band's own).  Returns (worst err/bar, failures [(key, band, err/bar)])."""
    worst, bad = 0.0, []
    for key, r in ref.items():
        g, e_ref = got[key].double().to(r.device), emu[key].to(r.device)
        if not torch.isfinite(g).all():
            bad.append((key, "whole", math.inf))
            continue
        regions = {"whole": (Ellipsis,)}
        if key.startswith("frame"):
            regions.update(frame_bands(*r.shape[2:]))
        for band, idx in regions.items():
            rb, gb, eb = r[idx], g[idx], e_ref[idx]
            m = rb.abs().max().item() if frame_max is None or not key.startswith("frame") else frame_max
            e, e_emu = (gb - rb).abs().max().item(), (eb - rb).abs().max().item()
            bar = k_emu(key) * e_emu + 1e-3 * m
            ratio = e / bar if bar > 0 else (0.0 if e == 0 else math.inf)
            worst = max(worst, ratio)
            if not e <= bar:
                bad.append((key, band, ratio))
    return worst, bad
