"""The guarded optimizer step without a device: the one-step-late step accounting (StepLedger), the loss-scale back-off
schedule, the constructor's checks, the record layout shared by the header and the binding, the argument checks of the
new entry points (every call here must fail before anything is launched), and that an optimizer with the guard off
reaches neither new entry point."""
import copy
import math
import os
import re
import subprocess
import tempfile

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rec(skip=False, sumsq=4.0, first_bad=-1, nonfinite=0):
    from bin_b200.optim import GradAudit
    if skip:
        nonfinite, first_bad = max(nonfinite, 1), max(first_bad, 0)
    return GradAudit(sumsq, nonfinite, first_bad, skip, math.sqrt(sumsq), 1.0)


class _Steps:
    """What Adam.step() does to its counters, minus the launches: advance at once, hand the ledger the way back."""

    def __init__(self, ledger):
        self.ledger, self.step, self.fetched = ledger, torch.tensor(0.0), 0

    def run(self, rec):
        self.ledger.resolve()
        seen = float(self.step)                        # the count the bias corrections of this step are built from
        self.step += 1

        def fetch():
            self.fetched += 1
            return rec
        self.ledger.submit(fetch, lambda: self.step.sub_(1))
        return seen


def test_ledger_applied_steps_advance_and_are_fetched_one_step_late():
    from bin_b200.optim import StepLedger
    led = StepLedger()
    s = _Steps(led)
    assert led.resolve() is None                       # nothing in flight, nothing resolved yet
    assert s.run(_rec()) == 0.0 and s.fetched == 0     # step() itself never waits for its own record
    assert s.run(_rec(sumsq=9.0)) == 1.0 and s.fetched == 1
    assert led.last.norm == 2.0                        # the record of step 1; step 2 is still in flight
    assert led.resolve().norm == 3.0 and s.fetched == 2
    assert led.resolve().norm == 3.0 and s.fetched == 2          # nothing in flight: the last record again, no wait
    assert float(s.step) == 2.0 and led.skipped_steps == 0


def test_ledger_skipped_step_does_not_advance():
    from bin_b200.optim import StepLedger
    led = StepLedger()
    s = _Steps(led)
    assert s.run(_rec()) == 0.0
    assert s.run(_rec(skip=True)) == 1.0
    assert float(s.step) == 2.0                        # counted as applied until it is resolved
    assert s.run(_rec()) == 1.0                        # the same bias corrections as the step that was skipped
    assert led.skipped_steps == 1
    assert s.run(_rec(skip=True)) == 2.0
    assert s.run(_rec(skip=True)) == 2.0               # twice in a row
    assert s.run(_rec()) == 2.0
    led.resolve()
    assert float(s.step) == 3.0 and led.skipped_steps == 3 and led.applied_run == 1


def test_ledger_refuses_two_steps_in_flight():
    from bin_b200.optim import StepLedger
    led = StepLedger()
    led.submit(lambda: _rec(), lambda: None)
    with pytest.raises(RuntimeError):
        led.submit(lambda: _rec(), lambda: None)


def test_backoff_schedule():
    from bin_b200.optim import BACKOFF_GROWTH_INTERVAL, LOSS_SCALE_MAX, StepLedger
    assert BACKOFF_GROWTH_INTERVAL == 1000 and LOSS_SCALE_MAX == 2048.0
    box = [2048.0]
    led = StepLedger((lambda: box[0], lambda x: box.__setitem__(0, x)))
    s = _Steps(led)
    for want in (1024.0, 512.0):
        s.run(_rec(skip=True))
        led.resolve()
        assert box[0] == want
    for _ in range(999):
        s.run(_rec())
    led.resolve()
    assert box[0] == 512.0
    s.run(_rec(skip=True))                             # a skip restarts the run of applied steps
    led.resolve()
    assert box[0] == 256.0
    for _ in range(1000):
        s.run(_rec())
    led.resolve()
    assert box[0] == 512.0
    for _ in range(3000):                              # the cap
        s.run(_rec())
    led.resolve()
    assert box[0] == 2048.0
    for _ in range(15):                                # the floor
        s.run(_rec(skip=True))
    led.resolve()
    assert box[0] == 1.0
    led2 = StepLedger()                                # without the option nothing is touched
    s2 = _Steps(led2)
    s2.run(_rec(skip=True))
    led2.resolve()
    assert led2.loss_scale is None


def test_loss_scale_target_accessors():
    from bin_b200 import autograd
    assert autograd.loss_scale_target() == autograd.LOSS_SCALE_TARGET == 2048.0
    try:
        autograd.set_loss_scale_target(64)
        assert autograd.loss_scale_target() == 64.0
        for bad in (0.5, 4096.0, float("nan")):
            with pytest.raises(ValueError):
                autograd.set_loss_scale_target(bad)
        assert autograd.loss_scale_target() == 64.0
    finally:
        autograd.set_loss_scale_target(autograd.LOSS_SCALE_TARGET)


def test_constructor_validation():
    from bin_b200.optim import Adam
    p = [torch.nn.Parameter(torch.zeros(3))]
    for bad in (0.0, -1.0, float("nan")):
        with pytest.raises(ValueError, match="max_grad_norm"):
            Adam(p, max_grad_norm=bad)
    with pytest.raises(ValueError, match="skip_nonfinite"):
        Adam(p, loss_scale_backoff=True)
    with pytest.raises(ValueError, match="skip_nonfinite"):
        Adam(p, max_grad_norm=1.0, loss_scale_backoff=True)
    opt = Adam(p, max_grad_norm=float("inf"), skip_nonfinite=True, loss_scale_backoff=True)
    assert opt.skipped_steps == 0 and opt.last_grad_norm is None and opt.last_nonfinite_param is None
    assert opt.resolve() is None
    plain = Adam(p)
    assert plain.max_grad_norm is None and not plain.skip_nonfinite and plain._ledger.loss_scale is None
    assert plain.state_dict()["state"] == {}


def test_state_dict_resolves_the_step_in_flight():
    """state_dict() after a skipped step that nobody has resolved yet: the saved `step` is the applied count, and the
    dict loads into torch.optim.Adam."""
    from bin_b200.optim import Adam
    p = torch.nn.Parameter(torch.zeros(3))
    opt = Adam([p], skip_nonfinite=True)
    step = torch.tensor(2.0)                            # two steps launched, the second still in flight
    opt.state[p].update(step=step, exp_avg=torch.zeros(3), exp_avg_sq=torch.zeros(3))
    opt._ledger.submit(lambda: _rec(skip=True), lambda: step.sub_(1))
    sd = opt.state_dict()
    assert float(sd["state"][0]["step"]) == 1.0 and opt.skipped_steps == 1
    ref = torch.optim.Adam([p])
    ref.load_state_dict(sd)
    assert float(ref.state[p]["step"]) == 1.0
    opt._ledger.submit(lambda: _rec(skip=True), lambda: step.sub_(1))
    opt.load_state_dict(copy.deepcopy(ref.state_dict()))   # loading resolves first: the old counter takes the skip, not the new
    assert float(step) == 0.0 and float(opt.state[p]["step"]) == 1.0 and opt.skipped_steps == 2


class _FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append(name)
            return 0
        return fn


def _fake_cuda_step(monkeypatch, **kw):
    """Adam.step() on CPU tensors that claim to be CUDA ones, against a library that records the calls."""
    import contextlib
    from bin_b200 import optim

    fake = _FakeLib()
    monkeypatch.setattr(optim, "lib", lambda: fake)
    monkeypatch.setattr(optim, "_stream", lambda: 0)
    monkeypatch.setattr(optim._Table, "__init__", lambda self, ps, ms, vs: self.__dict__.update(
        key=tuple(p.data_ptr() for p in ps) + tuple(m.data_ptr() for m in ms), params=list(ps), n=len(ps), nchunks=1,
        pkey=tuple(p.data_ptr() for p in ps),
        dev=torch.zeros(1), prefix=torch.zeros(1), ids=[], shared_step=None, step_value=0.0))
    monkeypatch.setattr(optim._Table, "upload", lambda self, grads: None)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    p = torch.nn.Parameter(torch.zeros(5))
    p.grad = torch.ones(5)
    opt = optim.Adam([p], **kw)
    return opt, p, fake


def test_default_step_reaches_neither_new_entry_point(monkeypatch):
    opt, p, fake = _fake_cuda_step(monkeypatch)
    opt.step()
    opt.step()
    assert fake.calls == ["bin_adam_step", "bin_adam_step"]
    assert float(opt.state[p]["step"]) == 2.0 and opt._ledger._in_flight is None


def test_layout_of_the_record_matches_the_header():
    """AUDIT_DTYPE (the view bin_b200.optim takes of the pinned record) == bin_grad_audit_t."""
    from bin_b200.optim import AUDIT_DTYPE
    fields = ["sumsq", "nonfinite", "first_bad", "skip", "norm", "coef"]
    assert list(AUDIT_DTYPE.names) == fields
    src = ['#include <stddef.h>', '#include <stdio.h>', '#include "bin_b200.h"', 'int main(void) {',
           '  printf("size %zu\\n", sizeof(bin_grad_audit_t));']
    src += [f'  printf("{f} %zu\\n", offsetof(bin_grad_audit_t, {f}));' for f in fields]
    src += ['  return 0;', '}']
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "a.c"), os.path.join(d, "a.out")
        open(c, "w").write("\n".join(src))
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = dict(line.split() for line in subprocess.check_output([exe], text=True).splitlines())
    assert int(got["size"]) == AUDIT_DTYPE.itemsize == 32
    for f in fields:
        assert int(got[f]) == AUDIT_DTYPE.fields[f][1], f


def test_new_symbols_are_declared_bound_and_leave_the_abi_version():
    from bin_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "bin_b200.h")).read()
    for name in ("bin_grad_audit_scratch_bytes", "bin_grad_audit", "bin_adam_step_guarded"):
        assert re.search(rf"\b{name}\s*\(", hdr) and name in _lib.exported_symbols()
    assert _lib.ABI_VERSION == 6


def test_entry_points_reject_bad_arguments_before_any_launch():
    from bin_b200 import _lib
    L = _lib.lib()
    inf = float("inf")
    assert L.bin_grad_audit_scratch_bytes(0) == 0 and L.bin_grad_audit_scratch_bytes(-3) == 0
    assert L.bin_grad_audit_scratch_bytes(2800) == 2800 * 16
    ok = dict(table=4096, prefix=4096, nt=1, nc=1, gs=1.0, mn=inf, scratch=4096, sb=16, rec=4096)

    def audit(**kw):
        a = dict(ok, **kw)
        return L.bin_grad_audit(a["table"], a["prefix"], a["nt"], a["nc"], a["gs"], a["mn"], a["scratch"], a["sb"],
                                a["rec"], None)
    ARG, WORKSPACE = 1, 4
    for kw in (dict(table=None), dict(prefix=None), dict(scratch=None), dict(rec=None), dict(nt=0), dict(nc=0),
               dict(mn=0.0), dict(mn=-1.0), dict(mn=float("nan")), dict(gs=inf), dict(gs=float("nan")),
               dict(scratch=4096 + 8), dict(rec=4096 + 4)):
        assert audit(**kw) == ARG, kw
        assert "grad_audit" in L.bin_last_error().decode()
    assert audit(sb=15) == WORKSPACE and audit(nc=3, sb=47) == WORKSPACE

    def guarded(table=4096, prefix=4096, nt=1, nc=1, bc1=0.1, bc2=0.01, rec=4096):
        return L.bin_adam_step_guarded(table, prefix, nt, nc, 1e-4, 0.9, 0.99, 1e-8, 0.0, bc1, bc2, 1.0, rec, None)
    for kw in (dict(table=None), dict(prefix=None), dict(rec=None), dict(rec=4096 + 4), dict(nt=0), dict(nc=0),
               dict(bc1=0.0), dict(bc2=0.0)):
        assert guarded(**kw) == ARG, kw
        assert "adam_step" in L.bin_last_error().decode()
