"""The restated learning-rate schemes (bin_b200.lr_scheduler, DESIGN §4s) against the reference's own
MultiStepLR_Restart, CosineAnnealingLR_Restart and BaseModel.update_learning_rate (tests/golden/lr_schedule.*, from
oracle/make_golden_lr.py): every iteration's lr of both groups bit for bit, the iterations a clear-state restart drops
the optimizer's state, and the state dicts.  Then a state dict round trip, a resume mid-schedule, and the train yml's
keys and refusals."""
import copy
import io
import json
import os
from collections import defaultdict

import numpy as np
import pytest
import torch

from bin_b200 import BinB200Error
from bin_b200 import train as T
from bin_b200.lr_scheduler import CosineAnnealingLR_Restart, MultiStepLR_Restart, warm_up
from oracle.make_golden_lr import jsonable
from test_train_driver_cpu import YML, with_

pytestmark = pytest.mark.filterwarnings("ignore:Detected call of")    # the loop steps the scheduler first, as intended


@pytest.fixture(scope="module")
def golden(golden_dir):
    with open(os.path.join(golden_dir, "lr_schedule.json")) as fh:
        meta = json.load(fh)["configs"]
    return meta, np.load(os.path.join(golden_dir, "lr_schedule.npz"))


class Resettable(torch.optim.SGD):
    """An optimizer with reset_state(), as optim.Adam has: records the scheduler step it was called at."""

    def __init__(self, params):
        super().__init__(params, lr=1.0)
        self.resets = []
        self.sched = None

    def reset_state(self):
        self.resets.append(self.sched.last_epoch)
        self.state = defaultdict(dict)


def _optimizer(cfg, kind):
    g = torch.Generator().manual_seed(5)
    p0, p1 = (torch.nn.Parameter(torch.randn(4, generator=g)) for _ in range(2))
    groups = [{"params": [p0], "lr": cfg["lrs"][0]}, {"params": [p1], "lr": cfg["lrs"][1]}]
    if kind == "adam":
        return torch.optim.Adam(groups, betas=(0.9, 0.99))
    return Resettable(groups)


def _scheduler(opt, cfg):
    kw = cfg["kwargs"]
    if cfg["scheme"] == "MultiStepLR":
        return MultiStepLR_Restart(opt, kw["milestones"], restarts=kw.get("restarts"), weights=kw.get("weights"),
                                   gamma=kw["gamma"], clear_state=kw["clear_state"])
    return CosineAnnealingLR_Restart(opt, kw["T_period"], restarts=kw.get("restarts"), weights=kw.get("weights"),
                                     eta_min=kw["eta_min"])


def _run(opt, sched, cfg, first, last, lrs, cleared, states=None):
    """update_learning_rate(k, warmup_iter) for k = first..last, as the trainer calls it before iteration k."""
    for k in range(first, last + 1):
        before = opt.state
        sched.step()
        warm_up(opt, k, cfg["warmup_iter"])
        if opt.state is not before:
            cleared.append(k)
        lrs[k - 1] = [g["lr"] for g in opt.param_groups]
        if states is not None and str(k) in cfg["states"]:
            states[str(k)] = jsonable(sched.state_dict())


NAMES = ["ms", "ms_no_clear", "ms_default_restart", "ms_warmup_before", "ms_warmup_past", "cos1", "cos3",
         "cos_default_restart", "cos_warmup_before", "cos_warmup_past"]


@pytest.mark.parametrize("kind", ["adam", "reset_state"])
@pytest.mark.parametrize("name", NAMES)
def test_schedule_equals_reference(golden, name, kind):
    meta, arrs = golden
    cfg = meta[name]
    opt = _optimizer(cfg, kind)
    sched = _scheduler(opt, cfg)
    if kind == "reset_state":
        opt.sched = sched
    states = {"0": jsonable(sched.state_dict())}
    lrs, cleared = np.zeros((cfg["iters"], 2)), []
    _run(opt, sched, cfg, 1, cfg["iters"], lrs, cleared, states)
    want = arrs[f"{name}_lr"]
    bad = np.nonzero(lrs.view(np.uint64) != want.view(np.uint64))
    assert bad[0].size == 0, [(int(i) + 1, int(j), lrs[i, j], want[i, j]) for i, j in zip(*bad)][:5]
    assert cleared == arrs[f"{name}_cleared"].tolist()
    if kind == "reset_state":                               # the optimizer's own reset, at the same iterations
        assert opt.resets == cleared
    assert states == cfg["states"]


@pytest.mark.parametrize("name,at", [("ms", 500), ("ms_warmup_past", 250), ("cos3", 600), ("cos_warmup_before", 50),
                                     ("cos1", 300)])
def test_resume_mid_schedule(golden, name, at):
    """The .state file's scheduler entry and the optimizer's groups, saved after iteration `at` and loaded into a new
    optimizer and scheduler, continue the sequence."""
    meta, arrs = golden
    cfg = meta[name]
    opt = _optimizer(cfg, "adam")
    sched = _scheduler(opt, cfg)
    lrs, cleared = np.zeros((cfg["iters"], 2)), []
    _run(opt, sched, cfg, 1, at, lrs, cleared)
    buf = io.BytesIO()
    torch.save({"schedulers": [sched.state_dict()], "optimizers": [opt.state_dict()]}, buf)
    buf.seek(0)
    saved = torch.load(buf)
    opt2 = _optimizer(dict(cfg, lrs=[0.5, 0.25]), "adam")   # other lrs: the loaded groups must win
    sched2 = _scheduler(opt2, cfg)
    opt2.load_state_dict(saved["optimizers"][0])
    sched2.load_state_dict(saved["schedulers"][0])
    assert jsonable(sched2.state_dict()) == jsonable(sched.state_dict())
    _run(opt2, sched2, cfg, at + 1, cfg["iters"], lrs, cleared)
    assert np.array_equal(lrs.view(np.uint64), arrs[f"{name}_lr"].view(np.uint64))
    assert cleared == arrs[f"{name}_cleared"].tolist()


def test_state_dict_round_trip():
    p = torch.nn.Parameter(torch.zeros(2))
    for make in (lambda o: MultiStepLR_Restart(o, [3, 3, 7], restarts=[5], weights=[0.5], gamma=0.5, clear_state=True),
                 lambda o: CosineAnnealingLR_Restart(o, [4, 6], restarts=[4], weights=[0.5], eta_min=1e-7)):
        a = make(torch.optim.SGD([p], lr=1e-4))
        for _ in range(6):
            a.step()
        b = make(torch.optim.SGD([p], lr=1e-4))
        b.load_state_dict(copy.deepcopy(a.state_dict()))
        assert jsonable(b.state_dict()) == jsonable(a.state_dict())
        assert T.scheduler_kind(a.state_dict()) == ("MultiStepLR" if isinstance(a, MultiStepLR_Restart)
                                                    else "CosineAnnealingLR_Restart")
    s = torch.optim.lr_scheduler.ReduceLROnPlateau(torch.optim.SGD([p], lr=1.0), "min", factor=0.2, patience=1)
    assert T.scheduler_kind(s.state_dict()) == "ReduceLROnPlateau"


def test_mismatched_restarts_raise_in_the_class():
    p = torch.nn.Parameter(torch.zeros(2))
    with pytest.raises(ValueError, match="differ in length"):
        MultiStepLR_Restart(torch.optim.SGD([p], lr=1.0), [2], restarts=[3, 5], weights=[1])


# ----------------------------------------------------------------------------- the yml
MS_YML = {"train.lr_scheme": "MultiStepLR", "train.lr_steps": [50000, 100000, 100000], "train.lr_gamma": 0.5,
          "train.restarts": [60000], "train.restart_weights": [0.5], "train.clear_state": True,
          "train.warmup_iter": 1000, "train.factor": None, "train.patience": None}
COS_YML = {"train.lr_scheme": "CosineAnnealingLR_Restart", "train.T_period": [250000, 250000, 250000],
           "train.eta_min": 1e-7, "train.restarts": [250000, 500000], "train.restart_weights": [1, 0.5],
           "train.factor": None, "train.patience": None}


def test_multistep_keys():
    o = T.parse_options(with_(**MS_YML))
    assert (o.lr_scheme, o.lr_steps, o.lr_gamma, o.restarts, o.restart_weights, o.clear_state, o.warmup_iter) == \
        ("MultiStepLR", [50000, 100000, 100000], 0.5, [60000], [0.5], True, 1000)
    assert (o.factor, o.patience, o.T_period, o.eta_min) == (None, None, None, None)
    o = T.parse_options(with_(**dict(MS_YML, **{"train.restarts": None, "train.restart_weights": None,
                                                "train.clear_state": None, "train.warmup_iter": None})))
    assert (o.restarts, o.restart_weights, o.clear_state, o.warmup_iter) == (None, None, False, -1)
    # factor and patience are read, and required, with ReduceLROnPlateau only
    assert T.parse_options(with_(**dict(MS_YML, **{"train.factor": 0.2}))).factor is None


def test_cosine_keys():
    o = T.parse_options(with_(**COS_YML))
    assert (o.lr_scheme, o.T_period, o.eta_min, o.restarts, o.restart_weights, o.warmup_iter) == \
        ("CosineAnnealingLR_Restart", [250000] * 3, 1e-7, [250000, 500000], [1.0, 0.5], -1)
    assert (o.lr_steps, o.lr_gamma, o.clear_state) == (None, None, False)
    o = T.parse_options(with_(**dict(COS_YML, **{"train.restarts": None, "train.restart_weights": None,
                                                 "train.T_period": [10, 20], "train.warmup_iter": 5})))
    assert (o.restarts, o.T_period, o.warmup_iter) == (None, [10, 20], 5)


def test_plateau_options_unchanged():
    """The shipped yml parses as before; the scheme keys take their defaults and are not read."""
    o = T.parse_options(YML)
    new = {"lr_scheme": "ReduceLROnPlateau", "lr_steps": None, "lr_gamma": None, "clear_state": False,
           "T_period": None, "eta_min": None, "restarts": None, "restart_weights": None, "warmup_iter": -1}
    assert {k: getattr(o, k) for k in new} == new
    assert T.Options(**{k: v for k, v in vars(o).items() if k not in new}) == o
    assert T.parse_options(with_(**{"train.warmup_iter": 10, "train.lr_steps": [5]})) == o
    with pytest.raises(BinB200Error, match=r"train\.factor is missing"):
        T.parse_options(with_(**{"train.factor": None}))


@pytest.mark.parametrize("over,key", [
    ({**MS_YML, "train.lr_steps": None}, "train.lr_steps"),
    ({**MS_YML, "train.lr_gamma": None}, "train.lr_gamma"),
    ({**MS_YML, "train.restart_weights": [0.5, 0.5]}, "train.restart_weights"),
    ({**MS_YML, "train.restarts": None, "train.restart_weights": [1, 1]}, "train.restarts"),
    ({**MS_YML, "train.lr_steps": 5000}, "train.lr_steps"),
    ({**COS_YML, "train.T_period": None}, "train.T_period"),
    ({**COS_YML, "train.eta_min": None}, "train.eta_min"),
    ({**COS_YML, "train.restart_weights": [1]}, "train.restart_weights"),
    ({**COS_YML, "train.T_period": [250000, 250000]}, "train.T_period"),
    ({**COS_YML, "train.restarts": None, "train.restart_weights": None, "train.T_period": [10]}, "train.T_period"),
    ({"train.lr_scheme": "StepLR"}, "train.lr_scheme"),
])
def test_refusals_name_key_and_scheme(over, key):
    with pytest.raises(BinB200Error) as e:
        T.parse_options(with_(**over))
    msg = str(e.value)
    assert key in msg and "train.lr_scheme" in msg, msg


def test_cosine_with_one_period_fails_in_the_reference_way():
    """What the T_period refusal prevents: with restarts unset, step 1 is a restart and reads T_period[1]."""
    p = torch.nn.Parameter(torch.zeros(2))
    s = CosineAnnealingLR_Restart(torch.optim.SGD([p], lr=1.0), [10], eta_min=0)
    with pytest.raises(IndexError):
        s.step()
