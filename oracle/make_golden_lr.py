"""Generate tests/golden/lr_schedule.npz and tests/golden/lr_schedule.json by EXECUTING THE REFERENCE'S OWN
models/lr_scheduler.py and BaseModel.update_learning_rate (models/base_model.py).

Run in the authoring container only (needs the reference checkout, at $BIN_REFERENCE or /root/reference):

    python oracle/make_golden_lr.py

Each configuration builds a dummy torch.optim.Adam with two parameter groups (lr 1e-4 and 3e-5), the reference's
scheduler on it, and a BaseModel whose `optimizers` / `schedulers` are those two; then, for iterations 1..N,
`update_learning_rate(k, warmup_iter)` runs before the (absent) step, as the trainer's loop calls it.  Stored:

* npz ``<name>_lr`` (N, 2) float64: each group's lr after update_learning_rate(k), i.e. the lr iteration k runs with;
  ``<name>_cleared``: the iterations at which the scheduler replaced ``optimizer.state`` (clear_state restarts).
* json: per configuration the scheme, its arguments, warmup_iter and N, and the scheduler's state_dict() after
  construction (key "0") and after chosen iterations, made JSON-safe by ``jsonable``.

Only these numbers enter the repository; nothing of the reference is copied.
"""
import importlib.util
import json
import os
import sys
from collections import Counter

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")
REF = os.environ.get("BIN_REFERENCE", "/root/reference")
N = 1000
LRS = (1e-4, 3e-5)
STATE_AT = (0, 1, 250, 251, 301, 501, 1000)

MS = dict(milestones=[100, 250, 250, 400, 650, 900], restarts=[500, 800], weights=[0.5, 0.25], gamma=0.5,
          clear_state=True)
COS1 = dict(T_period=[300, 300], restarts=[300], weights=[0.5], eta_min=1e-7)
COS3 = dict(T_period=[250, 250, 200, 150], restarts=[250, 500, 750], weights=[1, 0.5, 0.25], eta_min=1e-6)
CONFIGS = {
    # scheme, arguments, warmup_iter
    "ms": ("MultiStepLR", MS, -1),
    "ms_no_clear": ("MultiStepLR", dict(MS, clear_state=False), -1),
    "ms_default_restart": ("MultiStepLR", dict(milestones=[200, 400, 600, 800], gamma=0.1, clear_state=True), -1),
    "ms_warmup_before": ("MultiStepLR", MS, 60),
    "ms_warmup_past": ("MultiStepLR", MS, 300),
    "cos1": ("CosineAnnealingLR_Restart", COS1, -1),
    "cos3": ("CosineAnnealingLR_Restart", COS3, -1),
    "cos_default_restart": ("CosineAnnealingLR_Restart", dict(T_period=[400, 350], eta_min=0), -1),
    "cos_warmup_before": ("CosineAnnealingLR_Restart", COS3, 100),
    "cos_warmup_past": ("CosineAnnealingLR_Restart", COS1, 400),
}


def jsonable(v):
    """A scheduler state_dict as JSON-safe data: a Counter becomes {"Counter": [[key, count], ...]} in key order."""
    if isinstance(v, Counter):
        return {"Counter": [[k, c] for k, c in sorted(v.items())]}
    if isinstance(v, dict):
        return {str(k): jsonable(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return [jsonable(x) for x in v]
    return v


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    sys.path.insert(0, REF)
    ref_lr = _load("reference_lr_scheduler", os.path.join(REF, "models", "lr_scheduler.py"))
    ref_base = _load("reference_base_model", os.path.join(REF, "models", "base_model.py"))
    arrays, meta = {}, {}
    for name, (scheme, kw, warmup) in CONFIGS.items():
        g = torch.Generator().manual_seed(5)
        p0, p1 = (torch.nn.Parameter(torch.randn(4, generator=g)) for _ in range(2))
        opt = torch.optim.Adam([{"params": [p0], "lr": LRS[0]}, {"params": [p1], "lr": LRS[1]}],
                               betas=(0.9, 0.99))
        if scheme == "MultiStepLR":
            sched = ref_lr.MultiStepLR_Restart(opt, kw["milestones"], restarts=kw.get("restarts"),
                                               weights=kw.get("weights"), gamma=kw["gamma"],
                                               clear_state=kw["clear_state"])
        else:
            sched = ref_lr.CosineAnnealingLR_Restart(opt, kw["T_period"], restarts=kw.get("restarts"),
                                                     weights=kw.get("weights"), eta_min=kw["eta_min"])
        model = ref_base.BaseModel({"gpu_ids": None, "is_train": True})
        model.optimizers, model.schedulers = [opt], [sched]
        states = {"0": jsonable(sched.state_dict())}
        lrs, cleared = np.zeros((N, 2)), []
        for k in range(1, N + 1):
            before = opt.state
            before[p0]["seen"] = k                          # a stand-in for Adam's moments
            model.update_learning_rate(k, warmup_iter=warmup)
            if opt.state is not before:
                cleared.append(k)
            lrs[k - 1] = [grp["lr"] for grp in opt.param_groups]
            if k in STATE_AT:
                states[str(k)] = jsonable(sched.state_dict())
        arrays[f"{name}_lr"] = lrs
        arrays[f"{name}_cleared"] = np.array(cleared, dtype=np.int64)
        meta[name] = {"scheme": scheme, "kwargs": kw, "warmup_iter": warmup, "iters": N, "lrs": list(LRS),
                      "states": states}
    np.savez_compressed(os.path.join(GOLDEN, "lr_schedule.npz"), **arrays)
    with open(os.path.join(GOLDEN, "lr_schedule.json"), "w") as fh:
        json.dump({"source": "reference models/lr_scheduler.py and BaseModel.update_learning_rate, "
                             f"torch {torch.__version__}", "configs": meta}, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print("wrote lr_schedule.npz / lr_schedule.json:", {k: len(v) for k, v in arrays.items() if k.endswith("cleared")})


if __name__ == "__main__":
    main()
