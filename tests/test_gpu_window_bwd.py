"""The six-frame window's gradients against fp64, per tensor: autograd.window_apply (17 backbone calls in 4 batched
stages, 6 ConvLSTM cells, 14 outputs, frames read by stage 1 and again by stage 3) forward and backward on a light
window (net.model = RDN_residual_interp_5_input(lstm=True, GO=g0, D=d)) whose every backbone has no ReLU input near 0
on the calls the window makes of it (no_flip.no_flip_window_sd).

Each case is held to the bar of the whole-backbone tests (tests/no_flip.py): the 14 outputs within TOL_FP16 of fp64;
each gradient e <= k_emu e_emu + 1e-3 max|ref|, with e the CUDA error against the reference's own 20-call dataflow in
fp64 and e_emu the error of an oracle that runs the library's batched schedule with fp16 storage, so that it rounds the
gradients of all the calls of a stage at one scale, as bin_grad_scale does; the frame gradients' border bands again,
each band on its own, with the 1e-3 term taken of the largest frame gradient of the window (a frame read only by quiet calls
carries the absolute error of its stages' scale); every parameter of net.named_parameters() has its gradient; the "off"
growth channels' weights and biases get exactly 0.  The premise of the bar, no ReLU input near 0, is asserted on the
stage inputs the CUDA forward computed (in fp64 arithmetic), not only on the fp64 chain's: each stage's calls are
recorded by wrapping autograd.backbone_stage, which also pins the stage call counts 5 / 6 / 4 / 2.

Every case runs in the default mode, under torch.use_deterministic_algorithms(True) (whose NaN-filled torch.empty makes
a read of an unwritten element a non-finite gradient) and with set_activation_checkpointing(net, "recompute"); each mode
is held to the bar on its own.  The cotangents: c - 0.5 with c ~ U[0, 1) on all 14 outputs; on outputs 9 and 13 only
(the outputs of the last stage), where every other stage sees only gradient that came through later stages and the
ConvLSTM cells, so a stage mixes calls of very different sizes under one scale; on output 13 only, where o[5], o[6] and
o[8] reach the loss through ConvLSTM cells alone (so a cell backward that is 2^-6 off shows in model2_1 and model3_1,
where the other cases' direct cotangents drown it) and o[4] and o[7] not at all (calls whose output gradient is 0
beside calls whose is not); or the training loss, loss.pixel_loss(kind="l2") with its 3 cycle terms
against O.get_loss_6v2 in fp64 (L2: its gradient is smooth in the output, unlike L1's sign).
"""
import contextlib
import time

import pytest
import torch

from no_flip import BETA, CANON, check_gradients, check_no_relu_near_zero, no_flip_window_sd, window_oracle_grads
from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu
TOL_FP16 = 1e-3
STAGE_CALLS = (5, 6, 4, 2)


def _case(g0, d, B, H, W, cots="all", seed=0):
    return dict(g0=g0, d=d, B=B, H=H, W=W, cots=cots, seed=seed)


CASES = {
    "g64d1_34x62": _case(64, 1, 2, 34, 62, seed=1),          # h = 17, w = 31: conv-tile remainders
    "g64d2_h1": _case(64, 2, 1, 2, 62, seed=2),              # h = 1
    "g96d1_18x58": _case(96, 1, 2, 18, 58, seed=3),
    "final_only": _case(64, 2, 2, 18, 30, cots=(9, 13), seed=4),
    "o13_only": _case(64, 1, 1, 18, 30, cots=(13,), seed=4),
    "l2_loss": _case(64, 1, 2, 34, 62, cots="l2", seed=5),
    "g96d12": _case(96, 12, 1, 6, 30, seed=6),              # the shipped width and depth
}
MODES = ("default", "deterministic", "recompute")
_CACHE = {}
_T0 = []


@pytest.fixture(scope="module", autouse=True)
def _report():
    _T0.append(time.perf_counter())
    yield
    print(f"[window bwd] {time.perf_counter() - _T0[0]:.1f} s")


@contextlib.contextmanager
def _deterministic(on):
    """torch.use_deterministic_algorithms(on), with torch.empty filling new memory with NaN when on."""
    prev = torch.are_deterministic_algorithms_enabled(), torch.utils.deterministic.fill_uninitialized_memory
    torch.use_deterministic_algorithms(on, warn_only=True)
    torch.utils.deterministic.fill_uninitialized_memory = True
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev[0])
        torch.utils.deterministic.fill_uninitialized_memory = prev[1]


def _named(gfr, gp):
    return {**{f"frame{j}": g for j, g in enumerate(gfr)}, **gp}


def _oracle(name):
    """The case's frames, loss, no-flip window weights and the fp64 and emulating oracles' outputs and gradients."""
    if name in _CACHE:
        return _CACHE[name]
    _CACHE.clear()
    c = CASES[name]
    B, H, W, seed = c["B"], c["H"], c["W"], c["seed"]
    frames = O.synth_frames(6, B, H, W, seed=seed)
    targets = O.synth_frames(14, B, H, W, seed=seed + 1)
    if c["cots"] == "l2":
        gts64 = [t.to("cuda", torch.float64) for t in targets]
        cots = lambda outs: O.get_loss_6v2(outs, gts64, kind="l2")[0]
    else:
        cots = [t - 0.5 if c["cots"] == "all" or k in c["cots"] else None for k, t in enumerate(targets)]
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        sd = no_flip_window_sd(seed, c["g0"], c["d"], [f.to("cuda", torch.float64) for f in frames])
        ref_outs, gfr, gp = window_oracle_grads(frames, cots, sd, emulate=False)
        _, gfr_emu, gp_emu = window_oracle_grads(frames, cots, sd, emulate=True)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    ref, emu = _named(gfr, gp), _named(gfr_emu, gp_emu)
    frame_max = max(ref[f"frame{j}"].abs().max().item() for j in range(6))
    _CACHE[name] = dict(frames=frames, targets=targets, cots=cots, sd=sd, ref_outs=ref_outs, ref=ref, emu=emu,
                        frame_max=frame_max)
    return _CACHE[name]


def _net(c, sd):
    from bin_b200 import rdn
    net = rdn.bin_stage4_lstm()
    net.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=c["g0"], D=c["d"])
    net.load_state_dict(sd, strict=True)
    return net.cuda().train()


def _run(c, s, mode, monkeypatch):
    """One forward and backward of the window in `mode`: (outputs, {parameter or frame: gradient}, [(backbone name,
    the stage's calls)] as the forward ran them)."""
    from bin_b200 import autograd, loss, rdn
    net = _net(c, s["sd"])
    pyr = net.model
    names = {id(getattr(pyr, m)): m for m in CANON}
    stages = []
    real = autograd.backbone_stage

    def recording(model, calls):
        outs = real(model, calls)
        stages.append((names[id(model)], [[t.detach() for t in call] for call in calls]))
        return outs

    rdn.set_activation_checkpointing(net, "recompute" if mode == "recompute" else None)
    with monkeypatch.context() as mp, _deterministic(mode == "deterministic"):
        mp.setattr(autograd, "backbone_stage", recording)
        frg = [f.cuda().requires_grad_(True) for f in s["frames"]]
        outs = net(*frg)
        if c["cots"] == "l2":
            total = loss.pixel_loss(outs, [t.cuda() for t in s["targets"]], kind="l2")[0]
        else:
            total = sum((o * t.cuda()).sum() for o, t in zip(outs, s["cots"]) if t is not None)
        total.backward()
        torch.cuda.synchronize()
    grads = {k: p.grad for k, p in net.named_parameters()}
    grads.update({f"frame{j}": f.grad for j, f in enumerate(frg)})
    return [o.detach() for o in outs], grads, stages


def _group(key):
    if key.startswith("frame"):
        return "frames"
    return key.split(".")[1] if key.startswith("model.") else "clstm"


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(CASES))
def test_window_backward_vs_fp64(name, mode, monkeypatch):
    c = CASES[name]
    s = _oracle(name)
    outs, grads, stages = _run(c, s, mode, monkeypatch)

    # the premise of the bar, on the inputs the CUDA forward computed
    assert [(m, len(calls)) for m, calls in stages] == list(zip(CANON, STAGE_CALLS)), [(m, len(k)) for m, k in stages]
    margin = min(check_no_relu_near_zero([[t.double() for t in call] for call in calls],
                                         O.sub_sd(s["sd"], f"model.{m}"))[0] for m, calls in stages)

    fwd = max((o.double() - r).abs().max().item() for o, r in zip(outs, s["ref_outs"]))
    assert len(outs) == 14 and fwd <= TOL_FP16, (name, mode, fwd)

    d = c["d"]
    assert len(grads) == 6 + 4 * 2 * (5 * d + 6) + 12 and sorted(grads) == sorted(s["ref"])
    assert all(g is not None for g in grads.values()), [k for k, g in grads.items() if g is None]

    # the "off" channels' ReLU gradient is 0 everywhere: their growth weights and biases get exactly 0
    for m in CANON:
        for i in range(d):
            for cc in range(O.C):
                pre = f"model.{m}.RDBs.{i}.convs.{cc}.conv.0."
                off = (s["sd"][pre + "bias"] < 0).cuda()
                assert grads[pre + "weight"][off].abs().max().item() == 0.0, (pre, mode)
                assert grads[pre + "bias"][off].abs().max().item() == 0.0, (pre, mode)

    _, bad = check_gradients(grads, s["ref"], s["emu"], frame_max=s["frame_max"])
    per_group = {}
    for g in ("frames",) + CANON + ("clstm",):
        keys = [k for k in s["ref"] if _group(k) == g]
        per_group[g] = check_gradients({k: grads[k] for k in keys}, {k: s["ref"][k] for k in keys},
                                       {k: s["emu"][k] for k in keys}, frame_max=s["frame_max"])[0]
    print(f"[window bwd] {name} {mode}: forward {fwd:.1e}, ReLU margin on the CUDA inputs {margin / BETA:.3f} BETA, "
          "worst err/bar " + ", ".join(f"{g} {r:.3f}" for g, r in per_group.items()))
    assert not bad, sorted(bad, key=lambda r: -r[2])[:8]
