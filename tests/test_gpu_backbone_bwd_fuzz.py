"""Whole backbone backward launches against fp64, at the shapes, batches and call tables where the backward's glue goes
wrong: h or w of 1 and 2, tile multiples and remainders, maps that end on or one pixel past a 512-pixel p8_add /
p8_relu_mask group and a 1024-pixel p8_bias_grad block, 1 to 6 calls of 1 to 3 items, frames shared between slots and
calls, NULL frame gradients and unused outputs.

The glue kernels (grad_out_to_p8, pixel_unshuffle, p8_relu_mask, p8_add, p8_bias_grad and bias_grad_reduce,
unpack_frames_grad) and the launch table that chains them (plane offsets, workspace carve-up, call batching) have no
entry point of their own; they run only inside bin_backbone_bwd_masked / bin_backbone_bwd_recompute_masked.  So each
case runs autograd.backbone_stage forward and backward on weights with no ReLU input near 0 (tests/no_flip.py) and
holds it to fp64 autograd through oracle/arch_oracle.py with the bar of the whole-backbone tests: the forward within
TOL_FP16; each gradient e <= k_emu e_emu + 1e-3 max|ref|, where e_emu is the fp16-storage emulating oracle's error;
the frame gradients' last row and column and the rows and columns of the last conv tile again, each band on its own;
the "off" growth channels' weights and biases exactly 0.  Where some frames have no gradient, the deterministic run
also checks that every other gradient has the bits of a backward in which all frames want one.

Every case runs in the default mode and under torch.use_deterministic_algorithms(True), whose NaN-filled torch.empty
makes any read of an unwritten workspace element show up as a non-finite gradient; a third of them also recompute the
activations in the backward (set_activation_checkpointing(model, "recompute"), in deterministic mode).  Each mode is
held to the bar on its own.  Most cases are G0 in {64, 96} with D <= 3, whose fp64 oracle is cheap; the named D = 12
cases use small maps.

Cotangents.  The library scales all the calls of a launch by one power of two s, set by the loudest call
(s max|dOut| <= 2048, bin_grad_scale); the emulating oracle rounds each call's gradients with their own max.  The two
agree while the calls' cotangents are of one size, so every case keeps them within a factor of 2 of each other, except
"quiet", where call 1's cotangent is 2^-6 of the others.  That call's values are stored at the loud calls' scale, 64
times smaller than on their own.  fp16 keeps 11 significant bits from 2^-14 up, so this costs nothing until a value
drops under 2^-14; below that it keeps an absolute resolution of 2^-24 in scaled units, the floor the loud calls have
too.  So the quiet call's frame gradients carry the launch's absolute error, not one relative to their own size: their
1e-3 term is 1e-3 of the largest frame gradient of the launch (e <= k_emu e_emu + 1e-3 max over the launch's frames of
max|ref|), with e_emu still their own.  The weight gradients sum over the calls and keep the plain bar.
"""
import contextlib
import random
import statistics
import time

import pytest
import torch

from no_flip import BETA, check_gradients, check_no_relu_near_zero, no_flip_sd, oracle_grads
from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu
TOL_FP16 = 1e-3
CLASSES = {2: "RDN_residual_interp_2_input", 3: "RDN_residual_interp_2_1_input", 5: "RDN_residual_interp_4_1_input"}
HS = [1, 2, 3, 7, 8, 9, 16, 17, 33]                       # half-resolution h: 1, 2, around the 8-row conv tile
WS = [1, 2, 15, 29, 30, 31, 32, 33, 61, 64, 65]           # half-resolution w: around the 28-32-column conv tiles
QUIET = 2.0 ** -6


def _case(g0, d, n, ncalls, Bc, h, w, share="chain", nograd=(), unused=None, quiet=None, recompute=False, seed=0):
    return dict(g0=g0, d=d, n=n, ncalls=ncalls, Bc=Bc, h=h, w=w, share=share, nograd=tuple(nograd), unused=unused,
                quiet=quiet, recompute=recompute, seed=seed)


NAMED = {
    # the shipped width and depth, and the light width at full depth, at small maps
    "g96d12": _case(96, 12, 3, 2, 1, 3, 15, share="dup", recompute=True, seed=11),
    "g96d12_ncalls3": _case(96, 12, 2, 3, 1, 2, 33, seed=12),
    "g64d12": _case(64, 12, 5, 1, 2, 9, 31, recompute=True, seed=13),
    "g64d12_h1": _case(64, 12, 2, 2, 2, 1, 29, share="dup", seed=14),
    # h w at and one past a 512-pixel p8_add / p8_relu_mask group and a 1024-pixel p8_bias_grad block, and > 2048
    "hw512": _case(64, 1, 2, 1, 2, 16, 32, seed=21),
    "hw513": _case(64, 2, 3, 2, 1, 19, 27, recompute=True, seed=22),
    "hw1024": _case(96, 1, 2, 2, 1, 32, 32, seed=23),
    "hw1025": _case(64, 1, 5, 1, 2, 25, 41, seed=24),
    "hw2400": _case(64, 2, 2, 2, 2, 48, 50, recompute=True, seed=25),
    "many_tiles": _case(64, 1, 2, 1, 3, 72, 124, seed=26),           # more conv and wgrad tiles than SMs
    # call tables: BIN_MAX_CALLS = 6 calls of 3 items, the window's 5-call stage 1, the pyramid's sharing patterns
    "ncalls6_bc3": _case(64, 1, 2, 6, 3, 3, 5, seed=31),
    "ncalls6_bc3_n3": _case(96, 2, 3, 6, 3, 2, 7, share="dup", recompute=True, seed=32),
    "stage1_5calls": _case(64, 2, 2, 5, 1, 9, 31, seed=33),
    "stage2_dup": _case(64, 3, 3, 3, 1, 8, 30, share="dup", seed=34),                   # (I2, I2, I4) ...
    "stage4_dup": _case(96, 1, 5, 2, 2, 7, 29, share="dup", recompute=True, seed=35),  # (I4, I4, I4b, I6b, I6)
    # frames without a gradient (NULL dfr entries) between frames with one; an unused output (gout None -> zeros)
    "null_frames": _case(64, 2, 3, 3, 2, 9, 17, nograd=(1, 3), seed=41),
    "null_shared": _case(96, 1, 2, 4, 1, 17, 15, nograd=(2,), recompute=True, seed=42),
    "null_dup": _case(64, 1, 5, 2, 1, 8, 33, share="dup", nograd=(0,), seed=43),
    "unused": _case(64, 2, 2, 3, 2, 7, 30, unused=1, seed=44),
    "unused_null": _case(96, 1, 3, 4, 1, 16, 31, nograd=(0, 4), unused=3, recompute=True, seed=45),
    "quiet": _case(64, 2, 2, 3, 1, 17, 29, share="disjoint", quiet=1, seed=46),
    "h1w1": _case(64, 1, 2, 2, 3, 1, 1, seed=47),
    "h1w1_n5": _case(96, 1, 5, 3, 2, 1, 1, share="dup", recompute=True, seed=48),
}
NFUZZ = 27


def _draw(k):
    """Fuzz case k: h and w walk HS and WS (every value at least twice); the rest is drawn."""
    rnd = random.Random(9100 + k)
    h, w = HS[k % len(HS)], WS[k % len(WS)]
    while True:
        ncalls, Bc = rnd.randint(1, 6), rnd.randint(1, 3)
        if ncalls * Bc * h * w >= 4:          # the no-flip construction pools each channel over >= 4 values
            break
    n, share = rnd.choice([2, 3, 5]), rnd.choice(["chain", "chain", "dup", "disjoint"])
    c = _case(rnd.choice([64, 96]), rnd.randint(1, 3), n, ncalls, Bc, h, w, share=share, recompute=k % 3 == 0,
              seed=9100 + k)
    npool = len(_pool_index(c)[1])
    if npool > 1 and rnd.random() < 0.35:
        c["nograd"] = tuple(sorted(rnd.sample(range(npool), rnd.randint(1, max(1, npool // 3)))))
    if ncalls > 1 and rnd.random() < 0.25:
        c["unused"] = rnd.randrange(ncalls)
    return c


def _pool_index(c):
    """(pool size, calls_idx): chain = call k reads frames k .. k+n-2 and k+1 again (one tensor in two calls and, for
    n >= 3, in two slots of a call); dup = call k reads k, k, k+1 .. k+n-2 (stage 2 step 0 is (I2, I2, I4)); disjoint =
    each call its own n frames."""
    n, ncalls = c["n"], c["ncalls"]
    if c["share"] == "chain":
        idx = [list(range(k, k + n - 1)) + [k + 1] for k in range(ncalls)]
    elif c["share"] == "dup":
        idx = [[k, k] + list(range(k + 1, k + n - 1)) for k in range(ncalls)]
    else:
        idx = [list(range(n * k, n * k + n)) for k in range(ncalls)]
    return 1 + max(max(i) for i in idx), idx


def _id(name, c):
    return (f"{name}-g{c['g0']}d{c['d']}n{c['n']}-{c['h']}x{c['w']}-calls{c['ncalls']}-bc{c['Bc']}-{c['share']}"
            + ("-nullgrad" if c["nograd"] else "") + ("-unused" if c["unused"] is not None else "")
            + ("-quiet" if c["quiet"] is not None else ""))


CASES = {**NAMED, **{f"r{k}": _draw(k) for k in range(NFUZZ)}}
PARAMS = [pytest.param(name, mode, id=f"{_id(name, c)}-{mode}") for name, c in CASES.items()
          for mode in ("default", "deterministic") + (("recompute",) if c["recompute"] else ())]
RATIOS = {}
_CACHE = {}
_T0 = []


@pytest.fixture(scope="module", autouse=True)
def _report():
    _T0.append(time.perf_counter())
    yield
    for mode in sorted(RATIOS):
        r = sorted(RATIOS[mode])
        print(f"[backbone bwd fuzz] {mode:<13} cases {len(r):3d}  worst err/bar {r[-1]:.3f}  median {statistics.median(r):.3f}")
    print(f"[backbone bwd fuzz] {time.perf_counter() - _T0[0]:.1f} s")


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


def _oracle(name):
    """The case's frames, cotangents, no-flip weights and fp64 / fp16-storage oracle gradients, and its CUDA model."""
    if name in _CACHE:
        return _CACHE[name]
    _CACHE.clear()
    from bin_b200 import rdn
    c = CASES[name]
    n, ncalls, Bc, H, W, seed = c["n"], c["ncalls"], c["Bc"], 2 * c["h"], 2 * c["w"], c["seed"]
    npool, calls_idx = _pool_index(c)
    rnd = random.Random(seed)
    pool = O.synth_frames(npool, Bc, H, W, seed=seed)
    cots = []
    for k, t in enumerate(O.synth_frames(ncalls, Bc, H, W, seed=seed + 1)):
        t = t - 0.5
        t = t * (0.5 * rnd.uniform(0.55, 1.0) / t.abs().max())       # per-call max|dOut| within a factor of 2
        cots.append(None if k == c["unused"] else t * QUIET if k == c["quiet"] else t)
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        calls64 = [[pool[j].to("cuda", torch.float64) for j in idx] for idx in calls_idx]
        sd = {k: v.cpu() for k, v in no_flip_sd(n, seed, calls64, c["g0"], c["d"]).items()}
        margin, cv = check_no_relu_near_zero(calls64, sd)
        ref_outs, gfr, gp = oracle_grads(pool, calls_idx, cots, sd, emulate=False)
        _, gfr_emu, gp_emu = oracle_grads(pool, calls_idx, cots, sd, emulate=True)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    model = getattr(rdn, CLASSES[n])(G0=c["g0"], D=c["d"])
    model.load_state_dict(sd, strict=True)
    ref = {f"frame{j}": gfr[j] for j in range(npool) if j not in c["nograd"]}
    emu = {f"frame{j}": gfr_emu[j] for j in range(npool) if j not in c["nograd"]}
    ref.update(gp)
    emu.update(gp_emu)
    _CACHE[name] = dict(pool=pool, calls_idx=calls_idx, cots=cots, sd=sd, ref_outs=ref_outs, ref=ref, emu=emu,
                        model=model.cuda(), margin=margin, cv=cv)
    return _CACHE[name]


def _tiles_over_sms(Btot, h, w):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return Btot * -(-h // 8) * -(-w // 30) > sms and Btot * -(-h // 8) * -(-w // 16) > sms


def _run(s, nograd, mode):
    """One forward and backward of the case's model in `mode`: (outputs, {parameter or frame: gradient}), a frame at
    requires_grad False (in nograd) mapped to None."""
    from bin_b200 import autograd, rdn
    model = s["model"]
    model.zero_grad(set_to_none=True)
    rdn.set_activation_checkpointing(model, "recompute" if mode == "recompute" else None)
    try:
        with _deterministic(mode != "default"):
            frg = [p.cuda().requires_grad_(j not in nograd) for j, p in enumerate(s["pool"])]
            outs = autograd.backbone_stage(model, [[frg[j] for j in idx] for idx in s["calls_idx"]])
            sum((o * t.cuda()).sum() for o, t in zip(outs, s["cots"]) if t is not None).backward()
            torch.cuda.synchronize()
    finally:
        rdn.set_activation_checkpointing(model, None)
    grads = {k: p.grad for k, p in model.named_parameters()}
    grads.update({f"frame{j}": f.grad for j, f in enumerate(frg)})
    return [o.detach() for o in outs], grads


@pytest.mark.parametrize("name,mode", PARAMS)
def test_backbone_backward_vs_fp64(name, mode):
    c = CASES[name]
    s = _oracle(name)
    if name == "many_tiles":
        assert _tiles_over_sms(c["ncalls"] * c["Bc"], c["h"], c["w"])
    outs, grads = _run(s, c["nograd"], mode)
    fwd = max((o.double() - r).abs().max().item() for o, r in zip(outs, s["ref_outs"]))
    assert fwd <= TOL_FP16, (name, mode, fwd)
    assert all((grads[f"frame{j}"] is None) == (j in c["nograd"]) for j in range(len(s["pool"])))
    got = {k: grads[k] for k in s["ref"]}
    assert all(g is not None for g in got.values()), [k for k, g in got.items() if g is None]
    if c["nograd"] and mode == "deterministic":
        # a NULL frame gradient changes nothing else: every other gradient keeps the bits of the all-frames backward
        _, full = _run(s, (), mode)
        for k, g in got.items():
            assert torch.equal(g.view(torch.int32), full[k].view(torch.int32)), (k, "differs from the all-frames backward")
    frame_max = None
    if c["quiet"] is not None:
        frame_max = max(r.abs().max().item() for k, r in s["ref"].items() if k.startswith("frame"))
    worst, bad = check_gradients(got, s["ref"], s["emu"], frame_max=frame_max)
    # the "off" channels' ReLU gradient is 0 everywhere: their growth weights and biases get exactly 0
    for i in range(c["d"]):
        for cc in range(O.C):
            pre = f"RDBs.{i}.convs.{cc}.conv.0."
            off = (s["sd"][pre + "bias"] < 0).cuda()
            assert got[pre + "weight"][off].abs().max().item() == 0.0, (pre, mode)
            assert got[pre + "bias"][off].abs().max().item() == 0.0, (pre, mode)
    RATIOS.setdefault(mode, []).append(worst)
    print(f"[backbone bwd fuzz] {name} {mode}: forward {fwd:.1e}, worst gradient err/bar {worst:.3f} over {len(got)} "
          f"tensors, ReLU margin {s['margin'] / BETA:.3f} BETA, min std/mean {s['cv']:.3f}")
    assert not bad, sorted(bad, key=lambda r: -r[2])[:8]
