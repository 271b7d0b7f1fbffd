"""Multi-tensor Adam of the training step (SURVEY 8f rank 3).

`bin_model.__init__` builds `torch.optim.Adam(optim_params, lr=lr_G, weight_decay=wd_G, betas=(beta1, beta2))`
(bin_model.py:97-100) and `optimize_parameters` calls `.step()` after `l_pix.backward()` (:141).  `Adam` below is a
`torch.optim.Optimizer` with the same constructor, `param_groups` (the reference's schedulers write `group['lr']`,
lr_scheduler.py / bin_model.py:145) and per-parameter state (`step`, `exp_avg`, `exp_avg_sq` -- state dicts are
interchangeable with torch.optim.Adam, base_model.save_training_state), whose `step()` is ONE sm_90a launch per
parameter group over all tensors (`bin_adam_step`) instead of PyTorch's per-op foreach chain.

`Adam(..., max_grad_norm=x, skip_nonfinite=True)` guards the step (DESIGN §4i): one pass over all gradients on the
device (`bin_grad_audit`) finds their global norm and any inf or NaN, and `bin_adam_step_guarded` clips by that norm or
leaves every tensor untouched, without a host synchronisation.  `StepLedger` keeps the host's step count right.

CUDA fp32 parameters only; there is no CPU path."""
from __future__ import annotations

import logging
import math
from typing import Callable, Dict, List, NamedTuple, Optional, Tuple

import numpy as np
import torch

from ._lib import BinB200Error, check, lib

ADAM_CHUNK = 4096                                       # BIN_ADAM_CHUNK, include/bin_b200.h
AUDIT_DTYPE = np.dtype([("sumsq", "<f8"), ("nonfinite", "<u8"), ("first_bad", "<i4"), ("skip", "<i4"),
                        ("norm", "<f4"), ("coef", "<f4")])                     # bin_grad_audit_t
LOSS_SCALE_MAX = 2048.0                                 # autograd.LOSS_SCALE_TARGET
BACKOFF_GROWTH_INTERVAL = 1000                          # applied steps in a row that double the loss-scale target
_log = logging.getLogger(__name__)


class GradAudit(NamedTuple):
    """bin_grad_audit_t of one step as the host reads it.  `norm` is |grad_scale| * sqrt(sumsq) in fp64 (the device's
    record rounds it to fp32 to form `coef`); it and `sumsq` cover the finite elements."""
    sumsq: float
    nonfinite: int
    first_bad: int
    skip: bool
    norm: float
    coef: float


class StepLedger:
    """Host-side accounting of guarded steps, one step behind the device.  It knows nothing of CUDA.

    `step()` advances the step counters as if the step it launches will be applied, and hands the ledger `fetch`, which
    waits for that step's record, and `undo`, which takes the advance back.  `resolve()` runs them: at the start of the
    next `step()`, which needs the true count for its bias corrections, and before anything reads the counters
    (`state_dict()`).  A step found skipped leaves the count where torch would have it had the step never been tried.

    With `loss_scale` = (get, set) a skipped step halves the loss-scale target (floor 1) and BACKOFF_GROWTH_INTERVAL
    applied steps in a row double it (cap LOSS_SCALE_MAX)."""

    def __init__(self, loss_scale: Optional[Tuple[Callable[[], float], Callable[[float], None]]] = None):
        self.loss_scale = loss_scale
        self.skipped_steps = 0
        self.applied_run = 0
        self.last: Optional[GradAudit] = None
        self._in_flight: Optional[Tuple[Callable[[], GradAudit], Callable[[], None]]] = None

    def submit(self, fetch: Callable[[], GradAudit], undo: Callable[[], None]) -> None:
        if self._in_flight is not None:
            raise RuntimeError("StepLedger: resolve() the step in flight before submitting the next")
        self._in_flight = (fetch, undo)

    def resolve(self) -> Optional[GradAudit]:
        """The record of the step in flight, or of the last resolved step when none is (None before the first)."""
        if self._in_flight is None:
            return self.last
        (fetch, undo), self._in_flight = self._in_flight, None
        rec = self.last = fetch()
        if rec.skip:
            undo()
            self.skipped_steps += 1
            self.applied_run = 0
            if self.loss_scale:
                get, put = self.loss_scale
                put(max(1.0, get() / 2))
        else:
            self.applied_run += 1
            if self.loss_scale and self.applied_run == BACKOFF_GROWTH_INTERVAL:
                get, put = self.loss_scale
                put(min(LOSS_SCALE_MAX, get() * 2))
                self.applied_run = 0
        return rec


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


class _Table:
    """Device copy of the (p, g, m, v, n) table of one parameter group; only the gradient column changes per step
    (`zero_grad(set_to_none=True)` makes autograd hand out fresh gradient tensors)."""

    def __init__(self, params: List[torch.Tensor], ms: List[torch.Tensor], vs: List[torch.Tensor]):
        dev = params[0].device
        n = len(params)
        self.key = tuple(p.data_ptr() for p in params) + tuple(m.data_ptr() for m in ms)
        self.pkey = self.key[:n]
        self.params = list(params)
        self.host = torch.zeros((n, 5), dtype=torch.int64).pin_memory()
        h = self.host.numpy()
        h[:, 0] = [p.data_ptr() for p in params]
        h[:, 2] = [m.data_ptr() for m in ms]
        h[:, 3] = [v.data_ptr() for v in vs]
        h[:, 4] = [p.numel() for p in params]
        chunks = (h[:, 4] + ADAM_CHUNK - 1) // ADAM_CHUNK
        prefix = np.zeros(n + 1, dtype=np.int32)
        np.cumsum(chunks, out=prefix[1:])
        self.nchunks = int(prefix[-1])
        self.n = n
        self.prefix = torch.from_numpy(prefix).to(dev)
        self.dev = torch.empty((n, 5), dtype=torch.int64, device=dev)
        self.copied = torch.cuda.Event()
        self.ids: List[int] = []
        self.shared_step = None                         # one CPU tensor aliased by every state[p]["step"] of the group
        self.step_value = 0.0

    def upload(self, grads: List[torch.Tensor]) -> None:
        self.copied.synchronize()                       # the previous step's async copy has left the pinned buffer
        self.host.numpy()[:, 1] = [g.data_ptr() for g in grads]
        self.dev.copy_(self.host, non_blocking=True)
        self.copied.record()


class Adam(torch.optim.Optimizer):
    """torch.optim.Adam(params, lr, betas, eps, weight_decay) -- amsgrad / maximize / capturable are not offered
    (the reference does not use them).

    The guard is off by default, and `step()` then makes one `bin_adam_step` launch per parameter group.  Either of
    `max_grad_norm` (clip the gradients of all groups by their global L2 norm, as `clip_grad_norm_` over every
    parameter would) or `skip_nonfinite` turns it on: `step()` audits every gradient on the device and the step is
    skipped, for all groups, if one element is inf or NaN -- also with `max_grad_norm` alone, since the norm to clip by
    would not be finite.  `step()` never waits for the audit.  Its record is read one step late (`StepLedger`), or by
    `resolve()`, `state_dict()` and `load_state_dict()`, which do wait; `skipped_steps`, `last_grad_norm` and
    `last_nonfinite_param` describe the last resolved step.  Until a step is resolved, `state[p]["step"]` counts it as
    applied.

    A skipped step still bumps the parameters' `_version`: the next forward re-packs unchanged weights once, which is
    cheaper than the synchronisation that would avoid it.

    `loss_scale_backoff` (needs `skip_nonfinite`) also halves `autograd.loss_scale_target()` after each skipped step
    and doubles it after 1000 applied steps in a row, within [1, 2048].  The target is process-wide, and what moving
    it does to convergence has not been measured."""

    def __init__(self, params, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, max_grad_norm: Optional[float] = None, skip_nonfinite: bool = False,
                 loss_scale_backoff: bool = False):
        if lr < 0 or eps < 0 or weight_decay < 0 or not (0 <= betas[0] < 1 and 0 <= betas[1] < 1):
            raise ValueError("invalid Adam hyper-parameters")
        if max_grad_norm is not None and not max_grad_norm > 0:
            raise ValueError("max_grad_norm must be positive (or None)")
        if loss_scale_backoff and not skip_nonfinite:
            raise ValueError("loss_scale_backoff needs skip_nonfinite=True")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._tables: Dict[object, _Table] = {}           # (group, k), and "audit"
        self.max_grad_norm = None if max_grad_norm is None else float(max_grad_norm)
        self.skip_nonfinite = bool(skip_nonfinite)
        self.last_nonfinite_param: Optional[torch.Tensor] = None
        scale = None
        if loss_scale_backoff:
            from . import autograd
            scale = (autograd.loss_scale_target, autograd.set_loss_scale_target)
        self._ledger = StepLedger(scale)
        self._audit_bufs = None                        # (device record, pinned host record, event) of the guard

    @property
    def skipped_steps(self) -> int:
        return self._ledger.skipped_steps

    @property
    def last_grad_norm(self) -> Optional[float]:
        """Global L2 norm of the gradients of the last resolved step, before clipping (over the finite elements)."""
        return None if self._ledger.last is None else self._ledger.last.norm

    def resolve(self) -> Optional[GradAudit]:
        """Wait for the guarded step in flight and return its record (the last resolved one when none is in flight)."""
        return self._ledger.resolve()

    def state_dict(self):
        self.resolve()                                 # a saved `step` is exact
        sd = super().state_dict()
        # a `step` tensor of its own per parameter: torch.optim.Adam, stepping from this dict, adds 1 to each entry
        sd["state"] = {k: {**st, "step": st["step"].clone()} for k, st in sd["state"].items()}
        return sd

    def load_state_dict(self, state_dict):
        self.resolve()
        super().load_state_dict(state_dict)
        self._tables.clear()                           # exp_avg / exp_avg_sq / step tensors were replaced

    def add_param_group(self, param_group):
        if hasattr(self, "_tables"):
            self.resolve()
        super().add_param_group(param_group)
        if hasattr(self, "_tables"):
            self._tables.clear()

    def _launch(self, tab: _Table, group, step: float, grad_scale: float, audit: Optional[int]) -> None:
        beta1, beta2 = group["betas"]
        args = (tab.dev.data_ptr(), tab.prefix.data_ptr(), tab.n, tab.nchunks, float(group["lr"]), beta1, beta2,
                group["eps"], group["weight_decay"], 1.0 - beta1 ** step, 1.0 - beta2 ** step, grad_scale)
        with torch.cuda.device(tab.dev.device):
            if audit is None:
                check(lib().bin_adam_step(*args, _stream()))
            else:
                check(lib().bin_adam_step_guarded(*args, audit, _stream()))
        # The kernel writes the parameters through raw device pointers, which autograd's version counter does not see.
        # Every weight cache of the package (packed fp16 blobs, transposed blobs, the CUDA-graph key) is keyed on
        # (data_ptr, _version): without this bump the network would keep running on the weights packed BEFORE the step.
        torch._C._increment_version(tab.params)

    def _audit(self, launches, grad_scale: float) -> Tuple[int, Callable[[], GradAudit]]:
        """Audit the gradients of every launch into ONE device record.  Returns the record's device address, for the
        guarded launches that follow, and the ledger's `fetch` for this step."""
        if len(launches) == 1:
            tab = launches[0][0]
        else:                                          # one table over all groups: one norm, one decision
            ps = [p for t, _, _, _ in launches for p in t.params]
            ms = [self.state[p]["exp_avg"] for p in ps]
            tab = self._tables.get("audit")
            if tab is None or tab.key != tuple(p.data_ptr() for p in ps) + tuple(m.data_ptr() for m in ms):
                tab = self._tables["audit"] = _Table(ps, ms, [self.state[p]["exp_avg_sq"] for p in ps])
            tab.upload([g for _, gs, _, _ in launches for g in gs])
        dev = tab.dev.device
        if any(t.dev.device != dev for t, _, _, _ in launches):
            raise BinB200Error("bin_b200.optim.Adam: the gradient audit needs every parameter on one device")
        with torch.cuda.device(dev):
            if self._audit_bufs is None or self._audit_bufs[0].device != dev:
                self._audit_bufs = (torch.zeros(AUDIT_DTYPE.itemsize, dtype=torch.uint8, device=dev),
                                    torch.zeros(AUDIT_DTYPE.itemsize, dtype=torch.uint8).pin_memory(), torch.cuda.Event())
            rec_dev, rec_host, copied = self._audit_bufs
            scratch = torch.empty(lib().bin_grad_audit_scratch_bytes(tab.nchunks), dtype=torch.uint8, device=dev)
            check(lib().bin_grad_audit(tab.dev.data_ptr(), tab.prefix.data_ptr(), tab.n, tab.nchunks, grad_scale,
                                       math.inf if self.max_grad_norm is None else self.max_grad_norm,
                                       scratch.data_ptr(), scratch.numel(), rec_dev.data_ptr(), _stream()))
        params = tab.params

        def fetch() -> GradAudit:
            copied.synchronize()
            r = rec_host.numpy().view(AUDIT_DTYPE)[0]
            rec = GradAudit(float(r["sumsq"]), int(r["nonfinite"]), int(r["first_bad"]), bool(r["skip"]),
                            abs(grad_scale) * math.sqrt(float(r["sumsq"])), float(r["coef"]))
            self.last_nonfinite_param = params[rec.first_bad] if rec.skip else None
            if rec.skip:
                p = self.last_nonfinite_param
                _log.warning("bin_b200.optim.Adam: step skipped, %d non-finite gradient element(s); the first tensor "
                             "affected is parameter %d of the optimizer, shape %s", rec.nonfinite, rec.first_bad,
                             tuple(p.shape))
            return rec

        return rec_dev.data_ptr(), fetch

    @torch.no_grad()
    def step(self, closure=None, grad_scale: float = 1.0):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self.resolve()                                 # the bias corrections below need the number of APPLIED steps
        launches = []                                  # (table, gradients, group, step), launched after the loop
        advanced: List[torch.Tensor] = []              # the step counters this call advances ...
        shared: List[_Table] = []                      # ... and the tables that mirror theirs in step_value
        for gi, group in enumerate(self.param_groups):
            params = group["params"]
            grads = [p.grad for p in params]
            tab = self._tables.get((gi, 0))
            # steady state: same parameter objects as last step, every one with a dense contiguous gradient, one shared
            # step counter -> no per-tensor Python work beyond reading 540 gradient pointers
            if (tab is not None and tab.shared_step is not None and tab.ids == [id(p) for p in params]
                    and tab.pkey == tuple(p.data_ptr() for p in params)          # p.data re-homed (.to(), p.data = ...)?
                    and all(g is not None and g.is_contiguous() and g.dtype == torch.float32 and g.device == tab.dev.device
                            and not g.is_sparse for g in grads)):
                launches.append((tab, grads, group, float(tab.step_value) + 1.0))
                tab.shared_step += 1
                tab.step_value += 1
                advanced.append(tab.shared_step)
                shared.append(tab)
                continue
            by_step: Dict[float, List[torch.nn.Parameter]] = {}
            for p in params:
                if p.grad is None:
                    continue
                if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous()):
                    raise BinB200Error("bin_b200.optim.Adam: contiguous fp32 CUDA parameters only (no CPU path)")
                if p.grad.is_sparse or p.grad.dtype != torch.float32:
                    raise BinB200Error("bin_b200.optim.Adam: dense fp32 gradients only")
                st = self.state[p]
                if len(st) == 0:                       # torch/optim/adam.py _init_group
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                by_step.setdefault(float(st["step"]), []).append(p)
            for k, (step0, ps) in enumerate(by_step.items()):
                ms = [self.state[p]["exp_avg"] for p in ps]
                vs = [self.state[p]["exp_avg_sq"] for p in ps]
                gs = [p.grad if p.grad.is_contiguous() else p.grad.contiguous() for p in ps]
                key = tuple(p.data_ptr() for p in ps) + tuple(m.data_ptr() for m in ms)
                tab = self._tables.get((gi, k))
                if tab is None or tab.key != key:
                    tab = self._tables[(gi, k)] = _Table(ps, ms, vs)
                launches.append((tab, gs, group, step0 + 1.0))
                tab.ids, tab.shared_step = [id(p) for p in ps], None
                if len(by_step) == 1 and len(ps) == len(params):
                    # every tensor of the group is at the same step: let them share ONE counter tensor (state_dict()
                    # gives each parameter a copy)
                    tab.shared_step = torch.tensor(step0 + 1.0, dtype=torch.float32)
                    tab.step_value = step0 + 1.0
                    for p in ps:
                        self.state[p]["step"] = tab.shared_step
                    advanced.append(tab.shared_step)
                    shared.append(tab)
                else:
                    for p in ps:
                        self.state[p]["step"] = self.state[p]["step"] + 1
                        advanced.append(self.state[p]["step"])
        for tab, grads, _, _ in launches:
            with torch.cuda.device(tab.dev.device):
                tab.upload(grads)
        audit = fetch = None
        if launches and (self.skip_nonfinite or self.max_grad_norm is not None):
            audit, fetch = self._audit(launches, grad_scale)
        for tab, _, group, step in launches:
            self._launch(tab, group, step, grad_scale, audit)
        if audit is not None:
            rec_dev, rec_host, copied = self._audit_bufs
            with torch.cuda.device(rec_dev.device):
                rec_host.copy_(rec_dev, non_blocking=True)
                copied.record()

            def undo() -> None:
                for t in advanced:
                    t.sub_(1)
                for tab in shared:
                    tab.step_value -= 1
            self._ledger.submit(fetch, undo)
        return loss
