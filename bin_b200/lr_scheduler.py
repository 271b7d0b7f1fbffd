"""The reference's two restartable learning-rate schemes (models/lr_scheduler.py) and the linear warm-up of
BaseModel.update_learning_rate (models/base_model.py:51-63), restated for this package's trainer (DESIGN §4s).

Both schemes are chainable: an ordinary step derives the new lr from each group's current `lr`, so whatever else
wrote that lr (the warm-up, a user) carries into the schedule.  They compute in Python floats, with the reference's
order of operations, and give its bits.  Their state_dict() has the reference classes' keys and values, so a `.state`
file loads into either class.

A clear-state restart resets the optimizer: `optimizer.reset_state()` where it has one (`optim.Adam`), else the
reference's `optimizer.state = defaultdict(dict)`."""
from __future__ import annotations

import math
from collections import Counter, defaultdict
from typing import Optional, Sequence

from torch.optim.lr_scheduler import LRScheduler


def _restart_points(restarts: Optional[Sequence[int]], weights: Optional[Sequence[float]]):
    """-> (iterations, weights) of the restarts: an unset or empty list means one restart, at iteration 1, of weight 1.
    A restart given as r happens at scheduler step r + 1."""
    points = [r + 1 for r in (restarts or [0])]
    weights = list(weights or [1])
    if len(points) != len(weights):
        raise ValueError(f"restarts ({len(points)}) and restart_weights ({len(weights)}) differ in length")
    return points, weights


def _reset_optimizer(optimizer) -> None:
    reset = getattr(optimizer, "reset_state", None)
    if reset is not None:
        reset()
    else:
        optimizer.state = defaultdict(dict)


class MultiStepLR_Restart(LRScheduler):
    """lr_scheduler.MultiStepLR_Restart.  At a restart every group's lr becomes `initial_lr * weight` (and with
    `clear_state` the optimizer's state is dropped); at a milestone listed n times it is multiplied by gamma ** n;
    otherwise it is left as it is."""

    def __init__(self, optimizer, milestones, restarts=None, weights=None, gamma=0.1, clear_state=False,
                 last_epoch=-1):
        self.milestones = Counter(milestones)
        self.gamma = gamma
        self.clear_state = clear_state
        self.restarts, self.restart_weights = _restart_points(restarts, weights)
        super().__init__(optimizer, last_epoch)

    def get_lr(self):
        groups = self.optimizer.param_groups
        at = self.last_epoch
        if at in self.restarts:
            if self.clear_state:
                _reset_optimizer(self.optimizer)
            w = self.restart_weights[self.restarts.index(at)]
            return [g["initial_lr"] * w for g in groups]
        if at in self.milestones:
            decay = self.gamma ** self.milestones[at]
            return [g["lr"] * decay for g in groups]
        return [g["lr"] for g in groups]


class CosineAnnealingLR_Restart(LRScheduler):
    """lr_scheduler.CosineAnnealingLR_Restart, in its recursive form: each step scales `lr - eta_min` by the ratio of
    two consecutive points of the cosine of period T_max.  A restart sets the lr to `initial_lr * weight` and T_max
    to the next entry of T_period (so T_period needs one entry more than there are restarts).  Past T_max the curve
    continues: at T_max + 1 (mod 2 T_max) after a restart the step adds the cosine's first decrement, and the ratio
    then climbs back to the base lr."""

    def __init__(self, optimizer, T_period, restarts=None, weights=None, eta_min=0, last_epoch=-1):
        self.T_period = T_period
        self.T_max = self.T_period[0]
        self.eta_min = eta_min
        self.restarts, self.restart_weights = _restart_points(restarts, weights)
        self.last_restart = 0
        super().__init__(optimizer, last_epoch)

    def get_lr(self):
        groups = self.optimizer.param_groups
        at = self.last_epoch
        if at == 0:
            return list(self.base_lrs)
        if at in self.restarts:
            k = self.restarts.index(at)
            self.last_restart = at
            self.T_max = self.T_period[k + 1]
            return [g["initial_lr"] * self.restart_weights[k] for g in groups]
        t, T, lo = at - self.last_restart, self.T_max, self.eta_min
        if (t - 1 - T) % (2 * T) == 0:
            rise = 1 - math.cos(math.pi / T)
            return [g["lr"] + (base - lo) * rise / 2 for base, g in zip(self.base_lrs, groups)]
        ratio = (1 + math.cos(math.pi * t / T)) / (1 + math.cos(math.pi * (t - 1) / T))
        return [ratio * (g["lr"] - lo) + lo for g in groups]


def warm_up(optimizer, cur_iter: int, warmup_iter: int) -> None:
    """BaseModel.update_learning_rate's warm-up, after the scheduler's step of iteration `cur_iter` (1-based): while
    cur_iter < warmup_iter, every group's lr is `initial_lr / warmup_iter * cur_iter`."""
    if cur_iter < warmup_iter:
        for g in optimizer.param_groups:
            g["lr"] = g["initial_lr"] / warmup_iter * cur_iter
