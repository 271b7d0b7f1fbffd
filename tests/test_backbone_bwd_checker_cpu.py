"""The gradient bar of test_gpu_backbone_bwd_fuzz.py can fail: no_flip.check_gradients, fed fp64 gradients of a G0 = 64,
D = 1, two-frame backbone with one plausible indexing fault, rejects each of them, and accepts the fp16-storage
emulating oracle's gradients.  Each fault is applied both to the fp64 gradients and to the emulating oracle's, so the
bar has to tell it apart from fp16 storage error too."""
import pytest
import torch

from no_flip import check_gradients, check_no_relu_near_zero, no_flip_sd, oracle_grads
from oracle import bin_oracle as O

BIAS = "SFENet2.bias"


@pytest.fixture(scope="module")
def grads():
    n, seed, B, H, W = 2, 5, 1, 12, 20
    pool = O.synth_frames(n, B, H, W, seed=seed)
    calls_idx = [[0, 1]]
    cot = O.synth_frames(1, B, H, W, seed=seed + 1)[0] - 0.5
    calls = [[pool[j].double() for j in idx] for idx in calls_idx]
    sd = no_flip_sd(n, seed, calls, g0=64, d=1)
    check_no_relu_near_zero(calls, sd)
    _, gfr, gp = oracle_grads(pool, calls_idx, [cot], sd, emulate=False, device="cpu")
    _, gfr_emu, gp_emu = oracle_grads(pool, calls_idx, [cot], sd, emulate=True, device="cpu")
    ref = {"frame0": gfr[0], "frame1": gfr[1], **gp}
    emu = {"frame0": gfr_emu[0], "frame1": gfr_emu[1], **gp_emu}
    return ref, emu


def _last_col_zeroed(g):
    g["frame0"][..., -1] = 0


def _frames_swapped(g):
    g["frame0"], g["frame1"] = g["frame1"], g["frame0"]


def _bias_from_neighbour(g):
    g[BIAS][5] = g[BIAS][6]


def _last_row_shifted(g):
    g["frame1"][..., -1, :] = g["frame1"][..., -2, :]


FAULTS = {  # name: (fault, a (key, band) that must be among the failures)
    "last column zeroed": (_last_col_zeroed, ("frame0", "last col")),
    "frame slots swapped": (_frames_swapped, ("frame0", "whole")),
    "bias channel from its neighbour": (_bias_from_neighbour, (BIAS, "whole")),
    "last row shifted by one": (_last_row_shifted, ("frame1", "last row")),
}


def test_accepts_the_fp16_storage_oracle(grads):
    ref, emu = grads
    worst, bad = check_gradients(emu, ref, emu)
    assert not bad and worst <= 1.0 / 2.0, (worst, bad)   # e = e_emu: at most half the bar
    assert check_gradients(ref, ref, emu) == (0.0, [])


@pytest.mark.parametrize("base", ["fp64", "fp16-storage"])
@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_rejects_an_indexing_fault(grads, fault, base):
    ref, emu = grads
    fn, where = FAULTS[fault]
    got = {k: v.clone() for k, v in (ref if base == "fp64" else emu).items()}
    fn(got)
    _, bad = check_gradients(got, ref, emu)
    assert where in [(k, band) for k, band, _ in bad], bad
