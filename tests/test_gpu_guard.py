"""The guarded optimizer step on the GPU (DESIGN.md §4i): bin_grad_audit + bin_adam_step_guarded under
bin_b200.optim.Adam(max_grad_norm=..., skip_nonfinite=True).

Unless a test says otherwise the tensors are the 540 of bin_stage4_lstm() with seeded random gradients.  Non-finite
values are ordinary float data written into a gradient or an input frame."""
import copy
import hashlib
import logging
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HYPER = dict(lr=1e-4, betas=(0.9, 0.99), weight_decay=1e-5)


def _base_tensors():
    from bin_b200 import rdn
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(0), strict=True)
    ts = [p.detach().cuda() for p in m.parameters()]
    assert len(ts) == 540
    return ts


@pytest.fixture(scope="module")
def base():
    return _base_tensors()


def _params(base):
    return [torch.nn.Parameter(t.clone()) for t in base]


def _grads(ps, seed, scale=1e-2):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(p.shape, device="cuda", generator=g) * scale for p in ps]


def _give(ps, grads):
    for p, g in zip(ps, grads):
        p.grad = g.clone()


def _snapshot(opt, ps):
    torch.cuda.synchronize()
    return [(p.detach().clone(), opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone()) for p in ps]


def _same_bits(a, b):
    return [i for i, (x, y) in enumerate(zip(a, b)) if not all(torch.equal(u, v) for u, v in zip(x, y))]


def _norm64(grads):
    return math.sqrt(sum(float((g.double() ** 2).sum()) for g in grads))


# --------------------------------------------------------------------------------------------- 1. nothing is wrong
def test_guard_without_findings_writes_the_plain_step_bits(base):
    from bin_b200.optim import Adam
    ps, qs = _params(base), _params(base)
    guarded, plain = Adam(ps, skip_nonfinite=True, **HYPER), Adam(qs, **HYPER)
    for k in range(3):                                  # step 0 builds the table, 1-2 take the steady-state path
        grads = _grads(ps, 10 + k)
        _give(ps, grads)
        _give(qs, grads)
        guarded.step()
        plain.step()
    rec = guarded.resolve()
    assert not rec.skip and rec.nonfinite == 0 and rec.first_bad == -1 and rec.coef == 1.0
    assert _same_bits(_snapshot(guarded, ps), _snapshot(plain, qs)) == []
    assert all(float(guarded.state[p]["step"]) == float(plain.state[q]["step"]) == 3.0 for p, q in zip(ps, qs))
    assert guarded.skipped_steps == 0 and guarded.last_nonfinite_param is None


# --------------------------------------------------------------------------------------------- 2. the norm
def test_norm_matches_fp64_and_clip_grad_norm(base):
    from bin_b200.optim import Adam
    ps = _params(base)
    opt = Adam(ps, skip_nonfinite=True, **HYPER)
    grads = _grads(ps, 21)
    _give(ps, grads)
    opt.step()
    rec = opt.resolve()
    want = _norm64(grads)
    assert abs(opt.last_grad_norm - want) <= 1e-12 * want, (opt.last_grad_norm, want)
    assert rec.norm == opt.last_grad_norm and abs(rec.sumsq - want * want) <= 1e-12 * want * want
    ref = float(torch.nn.utils.clip_grad_norm_(ps, 1e30))
    assert abs(opt.last_grad_norm - ref) <= 1e-6 * ref, (opt.last_grad_norm, ref)
    opt.step(grad_scale=-0.5)                           # the norm is that of the gradients Adam sees
    assert abs(opt.resolve().norm - 0.5 * want) <= 1e-12 * want


def test_huge_finite_gradients_are_a_finite_norm_and_an_applied_step(base):
    """|g| ~ 1e25: an fp32 sum of squares would be inf and the step lost; the fp64 one clips it to max_grad_norm."""
    from bin_b200.optim import Adam
    ps = _params(base)
    opt = Adam(ps, max_grad_norm=1.0, **HYPER)
    grads = _grads(ps, 22, scale=1e25)
    _give(ps, grads)
    opt.step()
    rec = opt.resolve()
    want = _norm64(grads)
    assert math.isfinite(rec.norm) and abs(rec.norm - want) <= 1e-12 * want and want > 1e28
    assert not rec.skip and opt.skipped_steps == 0 and float(opt.state[ps[0]]["step"]) == 1.0
    assert 0 < rec.coef < 1e-27
    torch.cuda.synchronize()
    assert all(bool(torch.isfinite(p).all()) and bool(torch.isfinite(opt.state[p]["exp_avg_sq"]).all()) for p in ps)
    assert sum(not torch.equal(p.detach(), b) for p, b in zip(ps, base)) == 540


# --------------------------------------------------------------------------------------------- 3. clipping, exactly
def test_clipped_step_is_the_plain_step_scaled_by_coef(base):
    from bin_b200.optim import Adam
    ps, qs = _params(base), _params(base)
    max_norm = 0.5
    guarded, plain = Adam(ps, max_grad_norm=max_norm, **HYPER), Adam(qs, **HYPER)
    for k in range(2):
        grads = _grads(ps, 30 + k)
        _give(ps, grads)
        _give(qs, grads)
        guarded.step()
        rec = guarded.resolve()
        assert rec.norm > 10 * max_norm and 0 < rec.coef < 0.1
        want = np.float32(max_norm) / (np.float32(rec.norm) + np.float32(1e-6))
        assert abs(np.float32(rec.coef) - want) <= 2 * np.spacing(want), (rec.coef, want)
        plain.step(grad_scale=rec.coef)
        assert _same_bits(_snapshot(guarded, ps), _snapshot(plain, qs)) == []
    loose = Adam(_params(base), max_grad_norm=1e6, **HYPER)      # above the norm: nothing is clipped
    _give(loose.param_groups[0]["params"], grads)
    loose.step()
    assert loose.resolve().coef == 1.0


# --------------------------------------------------------------------------------------------- 4. skipping
def _skip_case(ps, qs, idx, elem, value):
    """One clean step on both, a step with `value` at gradient `idx`[`elem`] on the guarded one only, a clean step on
    both: the bad step leaves no trace."""
    from bin_b200.optim import Adam
    guarded, twin = Adam(ps, skip_nonfinite=True, **HYPER), Adam(qs, skip_nonfinite=True, **HYPER)
    grads = _grads(ps, 40)
    _give(ps, grads)
    _give(qs, grads)
    guarded.step()
    twin.step()
    before = _snapshot(guarded, ps)
    grads = _grads(ps, 41)
    grads[idx].view(-1)[elem] = value
    _give(ps, grads)
    guarded.step()
    rec = guarded.resolve()
    assert rec.skip and rec.nonfinite == 1 and rec.first_bad == idx
    assert _same_bits(_snapshot(guarded, ps), before) == []
    assert guarded.skipped_steps == 1 and guarded.last_nonfinite_param is ps[idx]
    assert all(float(guarded.state[p]["step"]) == 1.0 for p in ps)
    assert math.isfinite(guarded.last_grad_norm)
    grads = _grads(ps, 42)
    _give(ps, grads)
    _give(qs, grads)
    guarded.step()
    twin.step()
    assert not guarded.resolve().skip and guarded.last_nonfinite_param is None
    assert _same_bits(_snapshot(guarded, ps), _snapshot(twin, qs)) == []
    assert all(float(guarded.state[p]["step"]) == float(twin.state[q]["step"]) == 2.0 for p, q in zip(ps, qs))
    assert guarded.skipped_steps == 1 and twin.skipped_steps == 0


@pytest.mark.parametrize("value", [float("inf"), float("-inf"), float("nan")])
@pytest.mark.parametrize("where", ["first", "last"])
def test_one_nonfinite_element_skips_the_whole_step(base, where, value):
    idx, elem = (0, 0) if where == "first" else (539, -1)
    _skip_case(_params(base), _params(base), idx, elem, value)


@pytest.mark.parametrize("value", [float("inf"), float("-inf"), float("nan")])
@pytest.mark.parametrize("numel", [3, 4095, 4097])
@pytest.mark.parametrize("aligned", [False, True])
def test_nonfinite_last_element_of_small_and_odd_tensors(aligned, numel, value):
    """The scalar tails of a chunk and a second chunk of one element.  Unaligned: tensors cut from one flat buffer at
    odd offsets, which take the scalar path throughout; aligned: tensors of their own, vector loads plus a scalar tail."""
    sizes = [5, numel, 4096, 7]
    flat = torch.randn(sum(sizes) + 1, device="cuda", generator=torch.Generator(device="cuda").manual_seed(numel))

    def cut():
        f, out, o = flat.clone(), [], 1
        for n in sizes:
            out.append(torch.nn.Parameter(f[o:o + n].clone() if aligned else f[o:o + n]))
            o += n
        assert all((p.data_ptr() % 16 == 0) == aligned for p in out[:2])
        return out
    _skip_case(cut(), cut(), 1, numel - 1, value)


def test_skipped_step_is_logged_once_with_the_parameter(base, caplog):
    from bin_b200.optim import Adam
    ps = _params(base)
    opt = Adam(ps, skip_nonfinite=True, **HYPER)
    grads = _grads(ps, 43)
    grads[7].view(-1)[3] = float("nan")
    grads[300].view(-1)[0] = float("inf")
    _give(ps, grads)
    with caplog.at_level(logging.WARNING, logger="bin_b200.optim"):
        opt.step()
        rec = opt.resolve()
        opt.resolve()
    assert rec.nonfinite == 2 and rec.first_bad == 7
    msgs = [r.getMessage() for r in caplog.records if "step skipped" in r.getMessage()]
    assert len(msgs) == 1 and "parameter 7" in msgs[0] and str(tuple(ps[7].shape)) in msgs[0]


# --------------------------------------------------------------------------------------------- 5. two param groups
def test_two_param_groups_share_one_norm_and_one_decision(base):
    from bin_b200.optim import Adam
    cut = 500

    def groups(xs):                                     # bin_model.py:78-87: two groups, the first group's lr set later
        return [{"params": xs[:cut], "lr": 2e-4}, {"params": xs[cut:], "lr": 1e-4}]
    ps, qs = _params(base), _params(base)
    guarded, plain = Adam(groups(ps), max_grad_norm=0.5, **HYPER), Adam(groups(qs), **HYPER)
    grads = _grads(ps, 50)
    _give(ps, grads)
    _give(qs, grads)
    guarded.step()
    rec = guarded.resolve()
    want = _norm64(grads)
    assert abs(rec.norm - want) <= 1e-12 * want         # over both groups, not per group
    plain.step(grad_scale=rec.coef)
    assert _same_bits(_snapshot(guarded, ps), _snapshot(plain, qs)) == []
    before = _snapshot(guarded, ps)
    grads = _grads(ps, 51)
    grads[cut + 3].view(-1)[0] = float("nan")           # in the second group: the first must not move either
    _give(ps, grads)
    guarded.step()
    rec = guarded.resolve()
    assert rec.skip and rec.first_bad == cut + 3 and guarded.last_nonfinite_param is ps[cut + 3]
    assert _same_bits(_snapshot(guarded, ps), before) == []
    assert all(float(guarded.state[p]["step"]) == 1.0 for p in ps)


def test_frozen_parameters_stay_out_of_the_audit(base):
    from bin_b200.optim import Adam
    ps = _params(base)
    opt = Adam(ps, skip_nonfinite=True, **HYPER)
    grads = _grads(ps, 52)
    _give(ps, grads)
    for p in ps[:100]:
        p.grad = None
    opt.step()
    rec = opt.resolve()
    want = _norm64(grads[100:])
    assert not rec.skip and abs(rec.norm - want) <= 1e-12 * want
    torch.cuda.synchronize()
    assert all(torch.equal(p.detach(), b) for p, b in zip(ps[:100], base[:100])) and len(opt.state[ps[0]]) == 0


# --------------------------------------------------------------------------------------------- 6. determinism
def _record_bytes(tensors, stream=None, max_norm=0.5):
    """Raw bytes of the record bin_grad_audit leaves for seeded gradients (generated on the CPU: the same in any process)."""
    from bin_b200._lib import check, lib
    from bin_b200.optim import AUDIT_DTYPE, _Table
    g = torch.Generator().manual_seed(60)
    grads = [(torch.randn(t.shape, generator=g) * 1e-2).cuda() for t in tensors]
    grads[17].view(-1)[5] = float("inf")
    grads[400].view(-1)[0] = float("nan")
    torch.cuda.synchronize()
    with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream()):
        tab = _Table(tensors, tensors, tensors)         # the audit reads the g and n columns only
        tab.upload(grads)
        rec = torch.zeros(AUDIT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        scratch = torch.empty(lib().bin_grad_audit_scratch_bytes(tab.nchunks), dtype=torch.uint8, device="cuda")
        check(lib().bin_grad_audit(tab.dev.data_ptr(), tab.prefix.data_ptr(), tab.n, tab.nchunks, 1.0, max_norm,
                                   scratch.data_ptr(), scratch.numel(), rec.data_ptr(),
                                   torch.cuda.current_stream().cuda_stream))
        torch.cuda.current_stream().synchronize()
    return rec.cpu().numpy().tobytes()


def test_record_bytes_are_reproducible(base):
    from bin_b200.optim import AUDIT_DTYPE
    first = _record_bytes(base)
    r = np.frombuffer(first, dtype=AUDIT_DTYPE)[0]
    assert r["nonfinite"] == 2 and r["first_bad"] == 17 and r["skip"] == 1 and r["sumsq"] > 0
    assert all(_record_bytes(base) == first for _ in range(3))
    assert _record_bytes(base, stream=torch.cuda.Stream()) == first
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import test_gpu_guard as t\n"
            "print('RECORD', t._record_bytes(t._base_tensors()).hex())\n" % (ROOT, os.path.join(ROOT, "tests")))
    for cap in ("114", "66"):
        env = dict(os.environ, BIN_B200_MAX_SMS=cap)
        out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
        assert out.returncode == 0, out.stderr[-2000:]
        assert out.stdout.split("RECORD")[-1].strip() == first.hex(), cap


# --------------------------------------------------------------------------------------------- 7. end to end
def _train_net(mode=None):
    from bin_b200 import rdn
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(1), strict=True)
    return rdn.set_activation_checkpointing(m.cuda().train(), mode)


def _train_step(net, opt, fr, gt):
    from bin_b200.loss import pixel_loss
    opt.zero_grad(set_to_none=True)
    loss, _ = pixel_loss(net(*fr), gt, "l1")
    loss.backward()
    opt.step()
    return loss.detach()


def _digest(net):
    torch.cuda.synchronize()
    h = hashlib.sha256()
    for p in net.parameters():
        h.update(p.detach().cpu().numpy().tobytes())
    return h.hexdigest()


@pytest.mark.parametrize("mode", ["default", "recompute", "deterministic"])
def test_nan_pixel_skips_the_step_and_training_goes_on(mode):
    from bin_b200.optim import Adam
    B, H, W = 1, 64, 64
    fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=91, smooth=True)]
    gt = [f.cuda() for f in O.synth_frames(14, B, H, W, seed=92, smooth=True)]
    bad = [f.clone() for f in fr]
    bad[2][0, 1, 30, 31] = float("nan")
    torch.use_deterministic_algorithms(mode == "deterministic")
    try:
        net = _train_net("recompute" if mode == "recompute" else None)
        ps = list(net.parameters())
        opt = Adam(ps, lr=1e-4, betas=(0.9, 0.99), skip_nonfinite=True)
        _train_step(net, opt, fr, gt)                   # a clean step first, so that exp_avg / exp_avg_sq hold something
        before, state = _digest(net), _snapshot(opt, ps)
        _train_step(net, opt, bad, gt)
        rec = opt.resolve()
        assert rec.skip and rec.nonfinite > 0 and opt.skipped_steps == 1 and opt.last_nonfinite_param is ps[rec.first_bad]
        assert _digest(net) == before and _same_bits(_snapshot(opt, ps), state) == []
        assert all(float(opt.state[p]["step"]) == 1.0 for p in ps)
        l1 = _train_step(net, opt, fr, gt)
        assert not opt.resolve().skip and all(float(opt.state[p]["step"]) == 2.0 for p in ps)
        l2 = _train_step(net, opt, fr, gt)
        assert math.isfinite(float(l1)) and float(l2) < float(l1), (float(l1), float(l2))
        assert opt.skipped_steps == 1
    finally:
        torch.use_deterministic_algorithms(False)


# --------------------------------------------------------------------------------------------- 8. state dicts
def test_state_dict_round_trip_after_a_skipped_and_an_applied_step(base):
    from bin_b200.optim import Adam
    ps, qs = _params(base), _params(base)
    ours = Adam(ps, skip_nonfinite=True, **HYPER)
    for seed, poison in ((70, True), (71, False)):
        grads = _grads(ps, seed)
        if poison:
            grads[3].view(-1)[0] = float("nan")
        _give(ps, grads)
        ours.step()
    sd = copy.deepcopy(ours.state_dict())               # resolves the applied step still in flight
    assert ours.skipped_steps == 1 and all(float(s["step"]) == 1.0 for s in sd["state"].values())
    for q, p in zip(qs, ps):
        q.data.copy_(p.data)
    ref = torch.optim.Adam(qs, foreach=False, fused=False, **HYPER)
    ref.load_state_dict(sd)
    grads = _grads(ps, 72)
    _give(ps, grads)
    _give(qs, grads)
    ours.step()
    ref.step()
    worst = max(float((p.detach() - q.detach()).abs().max()) for p, q in zip(ps, qs))
    assert worst <= 2e-7, worst
    back = Adam(ps, skip_nonfinite=True, **HYPER)       # and back: torch's state into the guarded optimizer
    back.load_state_dict(copy.deepcopy(ref.state_dict()))
    grads = _grads(ps, 73)
    _give(ps, grads)
    _give(qs, grads)
    back.step()
    ref.step()
    assert not back.resolve().skip and float(back.state[ps[0]]["step"]) == float(ref.state[qs[0]]["step"]) == 3.0
    worst = max(float((p.detach() - q.detach()).abs().max()) for p, q in zip(ps, qs))
    assert worst <= 4e-7, worst


# --------------------------------------------------------------------------------------------- 9. loss-scale back-off
@pytest.mark.parametrize("backoff", [True, False])
def test_loss_scale_backoff(backoff):
    from bin_b200 import autograd
    from bin_b200.optim import Adam
    B, H, W = 1, 64, 64
    fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=93, smooth=True)]
    gt = [f.cuda() for f in O.synth_frames(14, B, H, W, seed=94, smooth=True)]
    bad = [f.clone() for f in fr]
    bad[0][0, 0, 5, 5] = float("nan")
    net = _train_net()
    opt = Adam(net.parameters(), lr=1e-4, betas=(0.9, 0.99), skip_nonfinite=True, loss_scale_backoff=backoff)
    assert autograd.loss_scale_target() == 2048.0
    try:
        _train_step(net, opt, bad, gt)
        assert autograd.loss_scale_target() == 2048.0   # not yet resolved
        l1 = _train_step(net, opt, fr, gt)              # resolves the skipped step on its way into step()
        after_skip = 1024.0 if backoff else 2048.0
        assert opt.skipped_steps == 1 and autograd.loss_scale_target() == after_skip
        l2 = _train_step(net, opt, fr, gt)              # this backward scaled its gradients to the halved target
        l3 = _train_step(net, opt, fr, gt)
        assert not opt.resolve().skip and opt.skipped_steps == 1
        assert autograd.loss_scale_target() == after_skip             # clean steps leave it alone
        assert all(math.isfinite(float(x)) for x in (l1, l2, l3))
    finally:
        autograd.set_loss_scale_target(autograd.LOSS_SCALE_TARGET)
