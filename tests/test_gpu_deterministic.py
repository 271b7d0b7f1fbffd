"""Deterministic training under torch.use_deterministic_algorithms(True) (DESIGN.md §4f).

With the flag on, the three cross-block sums that default to float atomicAdd -- the pixel-loss terms, the backbone bias
gradients and the ConvLSTM weight and bias gradients -- write one partial per block and add them in index order, and the
backbone weight gradients run on a constant grid of 132 CTAs instead of one per SM.  So a training step gives the same
bits from run to run, on any stream, in both activation-checkpointing modes and whatever SM count the library sees
(BIN_B200_MAX_SMS lowers the count the library uses for its grids, which is how one H100 stands in for smaller cards)."""
import hashlib
import os
import subprocess
import sys

import pytest
import torch

from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = (None, "recompute")


@pytest.fixture
def det():
    """Turn torch's deterministic mode on; restore it and the NaN fill of torch.empty afterwards."""
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(),
            torch.utils.deterministic.fill_uninitialized_memory)
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
    torch.utils.deterministic.fill_uninitialized_memory = prev[2]


@pytest.fixture(scope="module")
def net():
    from bin_b200 import rdn
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(0), strict=True)
    m = m.cuda().train()
    yield m
    rdn.set_activation_checkpointing(m, None)


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).abs() / b.abs().clamp_min(1e-30)).max().item()


def _close(a, b, rel):
    """max |a - b| within rel of the tensor's largest magnitude."""
    return (a.double() - b.double()).abs().max().item() <= rel * max(b.abs().max().item(), 1e-30)


def _is_conv_weight(name):
    return name.endswith(".weight") and ".Gates." not in name


def _sm_count_is_132():
    return torch.cuda.get_device_properties(0).multi_processor_count == 132 and not os.environ.get("BIN_B200_MAX_SMS")


# ---------------------------------------------------------------------------------------------------- pixel loss
def _loss_terms(outs, gts, kind):
    from bin_b200.loss import pixel_loss
    loss, ll = pixel_loss(outs, gts, kind)
    return loss, ll[0]._base                                 # all 17 pair terms (14 + 3 cycle terms)


def _fp64_terms(outs, gts, kind, eps=1e-6):
    from bin_b200.loss import CYCLE_PAIRS_6V2
    a = list(outs) + [outs[i] for i, _ in CYCLE_PAIRS_6V2]
    b = list(gts) + [outs[j] for _, j in CYCLE_PAIRS_6V2]
    terms = []
    for x, y in zip(a, b):
        d = (x.float() - y.float()).double()                # the kernel forms d in fp32
        t = d.abs().sum() if kind == "l1" else ((d * d).sum() if kind == "l2" else torch.sqrt(d * d + eps).mean())
        terms.append(t)
    return torch.stack(terms)


@pytest.mark.parametrize("n", [1, 1001, 3 * 64 * 96, 256 * 4096 * 2 + 3])
@pytest.mark.parametrize("kind", ["l1", "l2", "cb"])
def test_pixel_loss_bits(det, kind, n):
    g = torch.Generator(device="cuda").manual_seed(n + len(kind))
    outs = [torch.rand(n, device="cuda", generator=g) for _ in range(14)]
    gts = [torch.rand(n, device="cuda", generator=g) for _ in range(14)]
    runs = [_loss_terms(outs, gts, kind) for _ in range(5)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        runs.append(_loss_terms(outs, gts, kind))
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    loss0, terms0 = runs[0]
    assert terms0.numel() == 17
    for loss, terms in runs[1:]:
        assert torch.equal(loss, loss0) and torch.equal(terms, terms0)
    assert _rel(terms0, _fp64_terms(outs, gts, kind)) <= 1e-6
    torch.use_deterministic_algorithms(False)
    _, off = _loss_terms(outs, gts, kind)
    assert _rel(terms0, off) <= 1e-6


# ---------------------------------------------------------------------------------------------------- one backbone
BACKBONES = {2: "model1_1", 3: "model2_1", 5: "model3_1"}


def _backbone_grads(net, nframes, ncalls, B, H, W, mode):
    """One batched stage of `ncalls` calls, its backward for fixed cotangents; the backbone's parameter gradients."""
    from bin_b200 import rdn
    from bin_b200.autograd import backbone_stage
    model = getattr(net.model, BACKBONES[nframes])
    rdn.set_activation_checkpointing(net, mode)
    for p in model.parameters():
        p.grad = None
    frames = [f.cuda() for f in O.synth_frames(nframes * ncalls, B, H, W, seed=11 + nframes, smooth=True)]
    cots = [f.cuda() - 0.5 for f in O.synth_frames(ncalls, B, H, W, seed=12 + nframes)]
    outs = backbone_stage(model, [frames[k * nframes:(k + 1) * nframes] for k in range(ncalls)])
    torch.autograd.backward(outs, cots)
    torch.cuda.synchronize()
    rdn.set_activation_checkpointing(net, None)
    return {k: p.grad.clone() for k, p in model.named_parameters()}


def _max_bias_partials(ncalls, B, H, W):
    """Most block partials of any bias-gradient sum of one backward: blocks of 1024 px per item, at full resolution
    for UPNet.2 and at half resolution for the other convs."""
    per = lambda hw: ncalls * B * -(-hw // 1024)
    return max(per(H * W), per((H // 2) * (W // 2)))


# (nframes, calls, B, H, W): low-res wgrad tiles (16 x 8 px) per launch of 4 to 240, so some launches have fewer tiles
# than the 132-CTA grid and some more.  The 32 x 64 single calls have at most two partials per bias sum.
@pytest.mark.parametrize("nframes,ncalls,B,H,W", [(2, 1, 1, 32, 64), (5, 1, 1, 32, 64), (2, 1, 1, 48, 64),
                                                 (3, 6, 1, 64, 96), (5, 2, 2, 128, 160), (2, 3, 2, 128, 160)])
@pytest.mark.parametrize("mode", MODES)
def test_backbone_backward_bits(det, net, nframes, ncalls, B, H, W, mode):
    """Three repeats give the same bits.  Against the default mode: both add the same per-block partials v_j / scale
    (scale is a power of two, so dividing is exact), only in a different order.  With at most two partials the order
    cannot matter (fp32 addition is commutative), so the bias gradients must be bit-identical.  With P partials the
    two orders differ by at most 2 (P - 1) u sum|v_j| (u = 2^-24); at P <= 120 here that is below 1.42e-5 sum|v_j|,
    so the bar of 1e-3 of the tensor's largest gradient holds unless a channel's partials add up in magnitude to over
    70 times that gradient.  A misplaced or lost partial moves a bias gradient by a whole block's sum."""
    runs = [_backbone_grads(net, nframes, ncalls, B, H, W, mode) for _ in range(3)]
    assert len(runs[0]) == 132
    for r in runs[1:]:
        bad = [k for k in r if not torch.equal(r[k], runs[0][k])]
        assert not bad, bad[:8]
    torch.use_deterministic_algorithms(False)
    off = _backbone_grads(net, nframes, ncalls, B, H, W, mode)
    bias = [k for k in off if k.endswith(".bias")]
    assert len(bias) == 66
    if _max_bias_partials(ncalls, B, H, W) <= 2:
        bad = [k for k in bias if not torch.equal(runs[0][k], off[k])]
    else:
        bad = [k for k in bias if not _close(runs[0][k], off[k], 1e-3)]
    assert not bad, [(k, (runs[0][k] - off[k]).abs().max().item(), off[k].abs().max().item()) for k in bad[:8]]
    if _sm_count_is_132():                                   # the 132-CTA grid is the default grid on a full H100 SXM
        bad = [k for k in off if _is_conv_weight(k) and not torch.equal(runs[0][k], off[k])]
        assert not bad, bad[:8]


# ---------------------------------------------------------------------------------------------------- ConvLSTM
U32 = 2.0 ** -24                                             # unit roundoff of fp32


def _convlstm_bwd_abi(x, cp, hp, w, b, dh, dc, flags):
    """bin_convlstm_bwd_ex with the gate-gradient scratch in the caller's hands: returns (dw, db, dgates)."""
    from bin_b200 import _lib
    L = _lib.lib()
    B, _, H, W = x.shape
    dgates = torch.empty((B, 12, H, W), device="cuda")
    dx, dcp, dhp = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    dw, db = torch.zeros_like(w), torch.zeros_like(b)
    scratch = torch.empty(L.bin_convlstm_bwd_scratch_bytes(B, H, W), dtype=torch.uint8, device="cuda")
    P = lambda t: None if t is None else t.data_ptr()
    _lib.check(L.bin_convlstm_bwd_ex(x.data_ptr(), P(cp), P(hp), w.data_ptr(), b.data_ptr(), dh.data_ptr(), dc.data_ptr(),
                                     dgates.data_ptr(), dx.data_ptr(), P(dcp if cp is not None else None),
                                     P(dhp if hp is not None else None), dw.data_ptr(), db.data_ptr(), B, H, W, flags,
                                     scratch.data_ptr(), scratch.numel(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return dw, db, dgates


def _exact_weight_sums(x, hp, dgates):
    """fp64 sums of the kernel's own fp32 terms: dw[k][c][tap] = sum_p dgates[k][p] * in[c][p + tap] and db[k] =
    sum_p dgates[k][p] (every product of two fp32 values is exact in fp64), and the sums of their magnitudes."""
    inp = torch.cat((x, torch.zeros_like(x) if hp is None else hp), 1).double()
    inp = torch.nn.functional.pad(inp, (1, 1, 1, 1))
    g = dgates.double()
    H, W = x.shape[2], x.shape[3]
    dw, aw = torch.zeros((12, 6, 9), dtype=torch.float64, device="cuda"), torch.zeros((12, 6, 9), dtype=torch.float64, device="cuda")
    for t in range(9):
        ky, kx = divmod(t, 3)
        sl = inp[:, :, ky:ky + H, kx:kx + W]
        dw[:, :, t] = torch.einsum("bkyx,bcyx->kc", g, sl)
        aw[:, :, t] = torch.einsum("bkyx,bcyx->kc", g.abs(), sl.abs())
    return dw.reshape(12, 6, 3, 3), aw.reshape(12, 6, 3, 3), g.sum((0, 2, 3)), g.abs().sum((0, 2, 3))


@pytest.mark.parametrize("shape", [(2, 12, 14), (2, 96, 128)])
@pytest.mark.parametrize("with_state", [False, True])
def test_convlstm_weight_sums_within_the_rounding_bound(shape, with_state):
    """Both modes against the exact sum of the kernel's own terms.  Each output is a sum of its terms through at most
    n = L + 10 + P roundings: L pixels per lane, two 5-level shuffle trees and P block partials (the atomic path adds
    the P partials one after another; the deterministic reduce adds ceil(P/32) per lane).  Any such sum lies within
    gamma_n * sum|terms| of the exact one, gamma_n = n*u / (1 - n*u), so neither mode can fail this on correct code,
    whatever order the atomics take; the same bound, doubled, holds between the two modes."""
    B, H, W = shape
    sd = O.synth_state_dict(0)
    g = torch.Generator().manual_seed(5)
    x = torch.rand((B, 3, H, W), generator=g).cuda()
    cp = torch.randn((B, 3, H, W), generator=g).cuda() if with_state else None
    hp = torch.randn((B, 3, H, W), generator=g).tanh().cuda() if with_state else None
    dh, dc = torch.randn((B, 3, H, W), generator=g).cuda(), torch.randn((B, 3, H, W), generator=g).cuda()
    w = sd["clstm_5_prime_prime.Gates.weight"].cuda()
    b = sd["clstm_5_prime_prime.Gates.bias"].cuda()
    total = B * H * W
    P = min((total + 31) // 32, 592)
    n = -(-total // (P * 32)) + 10 + P
    gamma = n * U32 / (1 - n * U32)
    res = {}
    for flags in (0, 1):
        dw, db, dgates = _convlstm_bwd_abi(x, cp, hp, w, b, dh, dc, flags)
        ew, aw, eb, ab = _exact_weight_sums(x, hp, dgates)
        assert ((dw.double() - ew).abs() <= gamma * aw).all(), (flags, ((dw.double() - ew).abs() / aw).max().item(), gamma)
        assert ((db.double() - eb).abs() <= gamma * ab).all(), (flags, ((db.double() - eb).abs() / ab).max().item(), gamma)
        res[flags] = (dw, db, dgates)
    assert torch.equal(res[0][2], res[1][2])                  # the gate gradients are elementwise: same bits
    assert ((res[0][0].double() - res[1][0].double()).abs() <= 2 * gamma * aw).all()


@pytest.mark.parametrize("shape", [(2, 12, 14), (2, 96, 128)])
@pytest.mark.parametrize("with_state", [False, True])
def test_convlstm_backward_bits(det, net, shape, with_state):
    """Repeats give the same bits, and the result is within the fp32 backward's bar of an fp64 autograd through the
    oracle.  96 x 128 runs the weight-gradient kernel at its 592-block cap.  (The default mode's atomic sums vary from run
    to run by up to their rounding bound, so the two modes are compared against that bound, in the test above.)"""
    B, H, W = shape
    sd = O.synth_state_dict(0)
    g = torch.Generator().manual_seed(3)
    x = torch.rand((B, 3, H, W), generator=g)
    c0 = torch.randn((B, 3, H, W), generator=g)
    h0 = torch.randn((B, 3, H, W), generator=g).tanh()
    cot_h, cot_c = torch.randn((B, 3, H, W), generator=g), torch.randn((B, 3, H, W), generator=g)
    cell = net.clstm_5_prime_prime

    def run():
        cell.Gates.weight.grad = cell.Gates.bias.grad = None
        xg = x.clone().cuda().requires_grad_(True)
        stg = [t.clone().cuda().requires_grad_(True) for t in (c0, h0)] if with_state else None
        hh, (cc, _) = cell(xg, stg)
        ((hh * cot_h.cuda()).sum() + (cc * cot_c.cuda()).sum()).backward()
        torch.cuda.synchronize()
        return [xg.grad, cell.Gates.weight.grad.clone(), cell.Gates.bias.grad.clone()] + ([t.grad for t in stg] if stg else [])

    runs = [run() for _ in range(3)]
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(r, runs[0]))
    lsd = {k: v.double().requires_grad_(True) for k, v in sd.items() if k.startswith("clstm_5_prime_prime.")}
    xr = x.double().requires_grad_(True)
    st = tuple(t.double().requires_grad_(True) for t in (c0, h0)) if with_state else None
    h, (c, _) = O.convlstm(xr, lsd, "clstm_5_prime_prime", st)
    loss = (h * cot_h.double()).sum() + (c * cot_c.double()).sum()
    leaves = [xr, lsd["clstm_5_prime_prime.Gates.weight"], lsd["clstm_5_prime_prime.Gates.bias"]] + (list(st) if st else [])
    ref = torch.autograd.grad(loss, leaves)
    for a, b in zip(runs[0], ref):
        assert (a.cpu().double() - b).abs().max().item() <= 1e-4 * max(1.0, b.abs().max().item())


# ---------------------------------------------------------------------------------------------------- training steps
def _train(mode, steps=3, B=2, H=128, W=256):
    """`steps` Adam steps of the six-frame window from a fresh net (seed 0) with the Charbonnier loss; everything a
    step produces, and the weights and Adam state at the end."""
    from bin_b200 import rdn
    from bin_b200.loss import pixel_loss
    from bin_b200.optim import Adam
    torch.manual_seed(0)
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(1), strict=True)
    m = rdn.set_activation_checkpointing(m.cuda().train(), mode)
    opt = Adam(m.parameters(), lr=1e-4, betas=(0.9, 0.99))
    fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=21, smooth=True)]
    gt = [f.cuda() for f in O.synth_frames(14, B, H, W, seed=22, smooth=True)]
    out = []
    for _ in range(steps):
        opt.zero_grad(set_to_none=True)
        loss, ll = pixel_loss(m(*fr), gt, "cb")
        loss.backward()
        out.append((loss.detach().clone(), torch.stack(ll).detach().clone(),
                    {k: p.grad.clone() for k, p in m.named_parameters()}))
        opt.step()
    torch.cuda.synchronize()
    state = {k: v.clone() for k, v in m.state_dict().items()}
    adam = [(opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone()) for p in m.parameters()]
    return out, state, adam


def _assert_same_run(a, b):
    (sa, wa, ma), (sb, wb, mb) = a, b
    for k, ((la, lla, ga), (lb, llb, gb)) in enumerate(zip(sa, sb)):
        assert torch.equal(la, lb), ("loss", k, la.item(), lb.item())
        assert torch.equal(lla, llb), ("loss_list", k)
        assert len(ga) == len(gb) == 540
        bad = [n for n in ga if not torch.equal(ga[n], gb[n])]
        assert not bad, ("grads", k, bad[:8])
    bad = [n for n in wa if not torch.equal(wa[n], wb[n])]
    assert not bad, ("weights", bad[:8])
    assert len(ma) == len(mb) == 540
    assert all(torch.equal(x, y) for p, q in zip(ma, mb) for x, y in zip(p, q)), "Adam state"


def test_three_training_steps_bits(det):
    runs = {mode: [_train(mode) for _ in range(2)] for mode in MODES}
    for mode in MODES:
        _assert_same_run(*runs[mode])
    _assert_same_run(runs[None][0], runs["recompute"][0])     # bias and ConvLSTM gradients included
    losses = torch.stack([s[0] for s in runs[None][0][0]])
    assert (losses - losses[0]).abs().max().item() > 0      # the steps move the weights


# ---------------------------------------------------------------------------------------------------- SM count
_CHILD = r"""
import hashlib, sys, torch
sys.path.insert(0, %r)
from oracle import bin_oracle as O
from bin_b200 import rdn
from bin_b200.loss import pixel_loss
B, H, W = 2, 64, 96
net = rdn.bin_stage4_lstm(); net.load_state_dict(O.synth_state_dict(0), strict=True); net = net.cuda()
fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=31, smooth=True)]
gt = [f.cuda() for f in O.synth_frames(14, B, H, W, seed=32, smooth=True)]
def H_(ts):
    h = hashlib.sha256()
    for t in ts: h.update(t.detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()
def step():
    net.train(); net.zero_grad(set_to_none=True)
    f = [x.clone().requires_grad_(True) for x in fr]
    outs = net(*f)
    loss, ll = pixel_loss(outs, gt, "cb")
    loss.backward()
    return outs, loss, ll, dict(net.named_parameters()), f
torch.use_deterministic_algorithms(True)
outs, loss, ll, ps, f = step()
print("OUTS", H_(outs)); print("LOSS", H_([loss] + ll))
print("GRADS", H_([p.grad for p in ps.values()] + [x.grad for x in f]))
net.eval()
with torch.no_grad(): inf = net(*fr)
print("INFER", H_(inf))
torch.use_deterministic_algorithms(False)
outs, loss, ll, ps, f = step()
print("DEFAULT_WGRAD", H_([p.grad for k, p in ps.items() if k.endswith(".weight") and ".Gates." not in k]))
"""


def test_results_do_not_depend_on_the_sm_count():
    """One deterministic step and one inference window in children that see all SMs, 114 and 66 (the library reads
    BIN_B200_MAX_SMS once per process).  The default-mode conv weight gradients at 66 SMs must differ from those at the
    full count: that shows the knob reached the wgrad grid."""
    got = {}
    for tag in ("all", "114", "66"):
        env = {k: v for k, v in os.environ.items() if k != "BIN_B200_MAX_SMS"}
        if tag != "all":
            env["BIN_B200_MAX_SMS"] = tag
        r = subprocess.run([sys.executable, "-c", _CHILD % ROOT], env=env, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, (tag, r.stderr[-3000:])
        got[tag] = dict(line.split(" ", 1) for line in r.stdout.strip().splitlines() if line.split(" ", 1)[0].isupper())
        print("SMS", tag, got[tag])
    for key in ("OUTS", "LOSS", "GRADS", "INFER"):
        assert len({got[t][key] for t in got}) == 1, (key, {t: got[t][key] for t in got})
    if torch.cuda.get_device_properties(0).multi_processor_count > 66:
        assert got["66"]["DEFAULT_WGRAD"] != got["all"]["DEFAULT_WGRAD"]


# ---------------------------------------------------------------------------------------------------- unwritten memory
def _step_hashes(mode):
    from bin_b200 import rdn
    from bin_b200.loss import pixel_loss
    torch.manual_seed(0)
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(0), strict=True)
    m = rdn.set_activation_checkpointing(m.cuda().train(), mode)
    fr = [f.cuda().requires_grad_(True) for f in O.synth_frames(6, 2, 64, 96, seed=41, smooth=True)]
    gt = [f.cuda() for f in O.synth_frames(14, 2, 64, 96, seed=42, smooth=True)]
    outs = m(*fr)
    loss, ll = pixel_loss(outs, gt, "cb")
    loss.backward()
    ts = list(outs) + [loss] + ll + [p.grad for p in m.parameters()] + [f.grad for f in fr]
    assert len(ts) == 14 + 1 + 14 + 540 + 6
    bad = [k for k, t in enumerate(ts) if t is None or not torch.isfinite(t).all()]
    assert not bad, bad[:8]
    h = hashlib.sha256()
    for t in ts:
        h.update(t.detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


# 32-bit words left in freed memory: fp16 pairs (1.0, 1.0) / fp32 0.0078; fp16 pairs (57344, 57344) / fp32 6.6e35;
# fp16 pairs (0, -1.875) / fp32 -1.0.  All finite in both readings, so a kernel that read a byte it had not written
# would compute a finite but different result.
POISON = (0x3C003C00, 0x7B007B00, -0x40800000)


def _poison_allocator(word):
    """Fill the blocks the caching allocator hands out next with `word`: every workspace the step allocates with
    torch.empty then starts as that pattern (the fill of torch.empty is off)."""
    from bin_b200 import rdn
    rdn.release_workspaces()
    torch.cuda.empty_cache()
    big = torch.full(((torch.cuda.mem_get_info()[0] // 2) // 4,), word, dtype=torch.int32, device="cuda")
    small = [torch.full((1 << 17,), word, dtype=torch.int32, device="cuda") for _ in range(512)]
    torch.cuda.synchronize()
    del big, small


@pytest.mark.parametrize("mode", MODES)
def test_no_kernel_reads_unwritten_workspace(det, mode):
    """A deterministic step with the NaN fill on, then with it off after the allocator's free blocks were filled with
    each finite pattern of POISON: the outputs, loss and every gradient must be finite and hash the same every time."""
    from bin_b200 import rdn
    try:
        torch.utils.deterministic.fill_uninitialized_memory = True
        filled = _step_hashes(mode)
        torch.utils.deterministic.fill_uninitialized_memory = False
        for word in POISON:
            _poison_allocator(word)
            assert _step_hashes(mode) == filled, hex(word & 0xFFFFFFFF)
    finally:
        rdn.release_workspaces()
        torch.cuda.empty_cache()
