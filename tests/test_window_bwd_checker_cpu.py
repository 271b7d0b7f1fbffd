"""The window gradient bar of test_gpu_window_bwd.py can fail, and its oracles agree: on a G0 = 64, D = 1 window with no
ReLU input near 0 (no_flip.no_flip_window_sd), on a tiny map on the CPU,
- the library's batched schedule (bin_b200.rdn._window_schedule, each stage's calls concatenated along the batch) in
  fp64 gives the gradients of the reference's own 20-call dataflow (arch_oracle.window_forward) to 1e-12: the schedule
  is wired like the reference for gradients too;
- no_flip.check_gradients accepts the fp16-storage emulating oracle, and rejects each window-glue fault below, applied
  both to the fp64 gradients and to the emulating oracle's, so the bar has to tell it apart from fp16 storage error.

The faults, each with a (key, band) that must fail:
- "cell input detached": ConvLSTM cell 3 (clstm_5_prime_prime) reads o[5] without passing it a gradient; the
  h -> o[5] path is the window's quietest, so model2_1's UPNet.2 bias is what shows it;
- "stage 3 F[2] detached": stage 3's direct reads of frame 2 pass no gradient;
- "t2 detached": stage 4 reads t2 (stage 3's third call) for o[13] without passing it a gradient, which leaves cell 3
  (p5 -> t2) with no gradient;
- "stage 2 cotangents swapped": stage 2's first two calls (o[4], o[5]) get each other's output gradient; frame 0
  reaches the loss through o[0] and o[4] only.
"""
import pytest
import torch

from no_flip import check_gradients, no_flip_window_sd, window_oracle_grads
from oracle import bin_oracle as O

G0, D, B, H, W, SEED = 64, 1, 1, 6, 10, 3


def _named(r):
    _, gfr, gp = r
    return {**{f"frame{j}": g for j, g in enumerate(gfr)}, **gp}


@pytest.fixture(scope="module")
def window():
    frames = O.synth_frames(6, B, H, W, seed=SEED)
    sd = no_flip_window_sd(SEED, G0, D, [f.double() for f in frames])
    cots = [c - 0.5 for c in O.synth_frames(14, B, H, W, seed=SEED + 1)]
    run = lambda **kw: _named(window_oracle_grads(frames, cots, sd, device="cpu", **kw))
    ref, emu = run(emulate=False), run(emulate=True)
    frame_max = max(v.abs().max().item() for k, v in ref.items() if k.startswith("frame"))
    return run, ref, emu, frame_max


class _SwapGrad(torch.autograd.Function):
    """Identity on (a, b) whose backward hands a's gradient to b and b's to a."""

    @staticmethod
    def forward(ctx, a, b):
        return a.view_as(a), b.view_as(b)

    @staticmethod
    def backward(ctx, ga, gb):
        return gb, ga


def _cell_input_detached(stage, lstm, F):
    return stage, lambda group: lstm([(k, x.detach() if k == 3 else x) for k, x in group])


def _stage3_frame2_detached(stage, lstm, F):
    def st(name, calls):
        if name == "model3_1":
            calls = [[t.detach() if t is F[2] else t for t in c] for c in calls]
        return stage(name, calls)
    return st, lstm


def _t2_detached(stage, lstm, F):
    def st(name, calls):
        if name == "model4_1":
            calls = [calls[0], [t.detach() if j == 2 else t for j, t in enumerate(calls[1])]]
        return stage(name, calls)
    return st, lstm


def _stage2_cotangents_swapped(stage, lstm, F):
    def st(name, calls):
        outs = stage(name, calls)
        if name == "model2_1":
            outs[0], outs[1] = _SwapGrad.apply(outs[0], outs[1])
        return outs
    return st, lstm


FAULTS = {  # name: (fault, a (key, band) that must be among the failures)
    "cell input detached": (_cell_input_detached, ("model.model2_1.UPNet.2.bias", "whole")),
    "stage 3 F[2] detached": (_stage3_frame2_detached, ("frame2", "whole")),
    "t2 detached": (_t2_detached, ("clstm_5_prime_prime.Gates.weight", "whole")),
    "stage 2 cotangents swapped": (_stage2_cotangents_swapped, ("frame0", "whole")),
}


def test_batched_schedule_matches_the_reference_dataflow(window):
    run, ref, _, _ = window
    got = run(emulate=False, batched=True)
    assert sorted(got) == sorted(ref) and len(ref) == 6 + 4 * 2 * (5 * D + 6) + 12
    for k, r in ref.items():
        err = (got[k] - r).abs().max().item()
        assert err <= 1e-12 * r.abs().max().item(), (k, err, r.abs().max().item())


def test_accepts_the_fp16_storage_oracle(window):
    _, ref, emu, frame_max = window
    worst, bad = check_gradients(emu, ref, emu, frame_max=frame_max)
    assert not bad and worst <= 1.0 / 2.0, (worst, bad)   # e = e_emu: at most half the bar
    assert check_gradients(ref, ref, emu, frame_max=frame_max) == (0.0, [])


@pytest.mark.parametrize("base", ["fp64", "fp16-storage"])
@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_rejects_a_window_glue_fault(window, fault, base):
    run, ref, emu, frame_max = window
    fn, where = FAULTS[fault]
    got = run(emulate=base == "fp16-storage", batched=True, wrap=fn)
    _, bad = check_gradients(got, ref, emu, frame_max=frame_max)
    assert where in [(k, band) for k, band, _ in bad], sorted(bad, key=lambda r: -r[2])[:8]
