"""Multi-tensor Adam of the training step (SURVEY 8f rank 3).

`bin_model.__init__` builds `torch.optim.Adam(optim_params, lr=lr_G, weight_decay=wd_G, betas=(beta1, beta2))`
(bin_model.py:97-100) and `optimize_parameters` calls `.step()` after `l_pix.backward()` (:141).  `Adam` below is a
`torch.optim.Optimizer` with the same constructor, `param_groups` (the reference's schedulers write `group['lr']`,
lr_scheduler.py / bin_model.py:145) and per-parameter state (`step`, `exp_avg`, `exp_avg_sq` -- state dicts are
interchangeable with torch.optim.Adam, base_model.save_training_state), whose `step()` is ONE sm_90a launch per
parameter group over all tensors (`bin_adam_step`) instead of PyTorch's per-op foreach chain.

CUDA fp32 parameters only; there is no CPU path."""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np
import torch

from ._lib import BinB200Error, check, lib

ADAM_CHUNK = 4096                                       # BIN_ADAM_CHUNK, include/bin_b200.h


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
    (the reference does not use them)."""

    def __init__(self, params, lr: float = 1e-3, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0):
        if lr < 0 or eps < 0 or weight_decay < 0 or not (0 <= betas[0] < 1 and 0 <= betas[1] < 1):
            raise ValueError("invalid Adam hyper-parameters")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._tables: Dict[Tuple[int, int], _Table] = {}

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._tables.clear()                           # exp_avg / exp_avg_sq / step tensors were replaced

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        if hasattr(self, "_tables"):
            self._tables.clear()

    def _launch(self, tab: _Table, grads: List[torch.Tensor], group, step: float, grad_scale: float) -> None:
        beta1, beta2 = group["betas"]
        with torch.cuda.device(tab.dev.device):
            tab.upload(grads)
            check(lib().bin_adam_step(tab.dev.data_ptr(), tab.prefix.data_ptr(), tab.n, tab.nchunks,
                                      float(group["lr"]), beta1, beta2, group["eps"], group["weight_decay"],
                                      1.0 - beta1 ** step, 1.0 - beta2 ** step, grad_scale, _stream()))
        # The kernel writes the parameters through raw device pointers, which autograd's version counter does not see.
        # Every weight cache of the package (packed fp16 blobs, transposed blobs, the CUDA-graph key) is keyed on
        # (data_ptr, _version): without this bump the network would keep running on the weights packed BEFORE the step.
        torch._C._increment_version(tab.params)

    @torch.no_grad()
    def step(self, closure=None, grad_scale: float = 1.0):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
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
                self._launch(tab, grads, group, float(tab.step_value) + 1.0, grad_scale)
                tab.shared_step += 1
                tab.step_value += 1
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
                self._launch(tab, gs, group, step0 + 1.0, grad_scale)
                tab.ids, tab.shared_step = [id(p) for p in ps], None
                if len(by_step) == 1 and len(ps) == len(params):
                    # every tensor of the group is at the same step: let them share ONE counter tensor (state_dict()
                    # still shows a `step` per parameter; torch.save keeps the aliasing)
                    tab.shared_step = torch.tensor(step0 + 1.0, dtype=torch.float32)
                    tab.step_value = step0 + 1.0
                    for p in ps:
                        self.state[p]["step"] = tab.shared_step
                else:
                    for p in ps:
                        self.state[p]["step"] = self.state[p]["step"] + 1
        return loss
