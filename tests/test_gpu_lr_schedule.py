"""The restartable learning-rate schemes on the GPU (DESIGN §4s): optim.Adam's state reset -- by reset_state() and
by a reassigned `state`, eager, guarded and capturable with replays -- against a fresh Adam bit for bit and
torch.optim.Adam with its state cleared; then the driver with MultiStepLR and CosineAnnealingLR_Restart, warm-up and a
clear-state restart against a hand-written loop in the reference's call order, --cuda_graph against eager, resume
across a milestone and a restart, no host synchronisation, and two ranks when two GPUs are visible."""
import os
import random
import shutil
import socket
from collections import defaultdict

import pytest
import torch

from oracle import arch_oracle as A
from oracle import bin_oracle as O

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:Detected call of")]

SHAPES = [(96, 64, 3, 3), (96,), (5000,), (3, 7), (4096 * 3 + 5,)]
HYPER = dict(lr=1e-4, betas=(0.9, 0.99), weight_decay=1e-5)
RESET_AT = 3                                                # steps before the reset
AFTER = 3                                                   # steps after it


@pytest.fixture(autouse=True)
def _restore():
    yield
    torch.use_deterministic_algorithms(False)
    torch.utils.deterministic.fill_uninitialized_memory = True
    torch.cuda.set_sync_debug_mode(0)


# ----------------------------------------------------------------------------- 1. the optimizer's reset
def _params(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, device="cuda", generator=g) * 0.1) for s in SHAPES]


def _grads(seed, bad=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = [torch.randn(s, device="cuda", generator=g) * 1e-2 for s in SHAPES]
    if bad:
        out[1][3] = float("inf")
    return out


def _groups(ps, lr2=3e-5):
    return [{"params": ps[:3]}, {"params": ps[3:], "lr": lr2}]


def _set_grads(ps, gs, missing=()):
    for i, (p, g) in enumerate(zip(ps, gs)):
        if i in missing:
            p.grad = None
        elif p.grad is None:
            p.grad = g.clone()
        else:
            p.grad.copy_(g)                                 # capturable: the same gradient tensors every step


def _reset(opt, how):
    if how == "reset_state":
        opt.reset_state()
    else:
        opt.state = defaultdict(dict)                       # lr_scheduler.MultiStepLR_Restart(clear_state=True)


def _same(ps_a, opt_a, ps_b, opt_b):
    for a, b in zip(ps_a, ps_b):
        assert torch.equal(a, b)
        sa, sb = opt_a.state[a], opt_b.state[b]
        assert float(sa["step"]) == float(sb["step"])
        assert torch.equal(sa["exp_avg"], sb["exp_avg"]) and torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"])


class _Stepper:
    """Steps an Adam eagerly, or (capturable) eagerly once and then by replays of a graph that captured step()."""

    def __init__(self, opt, ps, graph):
        self.opt, self.ps, self.graph, self.g = opt, ps, graph, None

    def __call__(self, gs, missing=()):
        _set_grads(self.ps, gs, missing)
        if self.g is not None:
            self.opt.replay(self.g)
            return
        self.opt.step()
        if self.graph:
            self.g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.g):
                self.opt.step()


@pytest.mark.parametrize("how", ["reset_state", "assign"])
@pytest.mark.parametrize("mode", ["eager", "eager_grouped", "guarded", "guarded_skip", "capturable", "capturable_guarded"])
def test_reset_equals_fresh_adam(mode, how):
    """3 steps, a reset, 3 more: after the reset the parameters, moments and step counts equal a fresh Adam's built on
    the parameters at the reset, step after step, and stay within 2e-7 of torch.optim.Adam whose state was cleared at
    the same point.  eager_grouped: one parameter has no gradient at step 1, so the steps before the reset run the
    per-step grouping path; guarded_skip: the step just before the reset is skipped (an inf gradient) and still in
    flight when the reset comes."""
    from bin_b200.optim import Adam
    capturable = mode.startswith("capturable")
    guard = dict(skip_nonfinite=True) if "guarded" in mode else {}
    if mode == "capturable_guarded":
        guard["max_grad_norm"] = 1e3
    ps = _params(1)
    opt = Adam(_groups(ps), capturable=capturable, **guard, **HYPER)
    ref_ps = _params(1)
    ref = torch.optim.Adam(_groups(ref_ps), foreach=False, **HYPER)
    run = _Stepper(opt, ps, capturable)
    for k in range(RESET_AT):
        gs = _grads(10 + k, bad=(mode == "guarded_skip" and k == RESET_AT - 1))
        missing = (4,) if mode == "eager_grouped" and k == 0 else ()
        run(gs, missing)
        if not (mode == "guarded_skip" and k == RESET_AT - 1):
            _set_grads(ref_ps, gs, missing)
            ref.step()
    skipped = opt.skipped_steps if mode != "guarded_skip" else None
    fresh_ps = [torch.nn.Parameter(p.detach().clone()) for p in ps]
    fresh = Adam(_groups(fresh_ps), capturable=capturable, **guard, **HYPER)
    if capturable:
        keep = {id(p): (opt.state[p]["exp_avg"].data_ptr(), opt.state[p]["exp_avg_sq"].data_ptr()) for p in ps}
    _reset(opt, how)
    ref.state = defaultdict(dict)
    for k in range(AFTER):
        gs = _grads(20 + k)
        run(gs)
        _set_grads(fresh_ps, gs)
        fresh.step()
        _set_grads(ref_ps, gs)
        ref.step()
        _same(ps, opt, fresh_ps, fresh)
        assert float(opt.state[ps[0]]["step"]) == k + 1
    if capturable:                                          # the graph's tensors, bound to the new state
        assert run.g is not None
        assert all(keep[id(p)] == (opt.state[p]["exp_avg"].data_ptr(), opt.state[p]["exp_avg_sq"].data_ptr())
                   for p in ps)
    if mode == "guarded_skip":
        assert opt.skipped_steps == 1
    elif guard:
        opt.resolve()
        assert opt.skipped_steps == skipped == 0
    sd, sf = opt.state_dict(), fresh.state_dict()
    assert sd["param_groups"] == sf["param_groups"]
    for i in sd["state"]:
        for n in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(sd["state"][i][n].cpu(), sf["state"][i][n].cpu()), (i, n)
    worst = max(float((a.detach() - b.detach()).abs().max()) for a, b in zip(ps, ref_ps))
    assert worst <= 2e-7, worst


def test_capturable_reset_keeps_the_device_skip_count():
    """A replay skipped before the reset stays counted after it; the step count restarts from 0."""
    from bin_b200.optim import Adam
    ps = _params(2)
    opt = Adam(_groups(ps), capturable=True, skip_nonfinite=True, **HYPER)
    run = _Stepper(opt, ps, True)
    run(_grads(1))
    run(_grads(2, bad=True))
    opt.reset_state()
    run(_grads(3))
    opt.resolve()
    assert opt.skipped_steps == 1 and float(opt.state[ps[0]]["step"]) == 1.0


def test_reset_inside_a_capture_is_refused():
    from bin_b200 import BinB200Error
    from bin_b200.optim import Adam
    ps = _params(3)
    opt = Adam(_groups(ps), capturable=True, **HYPER)
    _set_grads(ps, _grads(1))
    opt.step()
    opt.state = defaultdict(dict)
    g = torch.cuda.CUDAGraph()
    with pytest.raises(BinB200Error, match="reset"):
        with torch.cuda.graph(g):
            opt.step()


# ----------------------------------------------------------------------------- 2. the driver
MS = {"train.lr_scheme": "MultiStepLR", "train.lr_steps": [2, 5, 5], "train.lr_gamma": 0.5, "train.restarts": [3],
      "train.restart_weights": [0.5], "train.clear_state": True, "train.warmup_iter": 3}
COS = {"train.lr_scheme": "CosineAnnealingLR_Restart", "train.T_period": [3, 4], "train.restarts": [2],
       "train.restart_weights": [0.5], "train.eta_min": 1e-6, "train.warmup_iter": 2}
SCHEMES = {"ms": MS, "cos": COS}


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    from test_gpu_train_driver import make_tree
    root = tmp_path_factory.mktemp("lr_tree")
    tree = str(root / "blur")
    make_tree(tree, "train", ["clipA", "clipB", "clipC"], 1)
    make_tree(tree, "test", ["clipV"], 2)
    weights = {}
    for name, sd in (("shipped", O.synth_state_dict(0)), ("light", A.synth_state_dict(0, 64, 6))):
        weights[name] = str(root / f"{name}.pth")
        torch.save(sd, weights[name])
    return tree, weights


def _options(tree, save, weights, scheme, **over):
    from test_gpu_train_driver import options
    opt = options(tree, save, weights, **over)
    for k in ("factor", "patience"):
        opt["train"].pop(k)
    for k, v in SCHEMES[scheme].items():
        opt["train"][k.split(".", 1)[1]] = v
    return opt


def _driver(opt, iters, **kw):
    from bin_b200 import train as T
    t = T.Trainer(T.parse_options(opt), deterministic=True, stdout=False, **kw)
    try:
        t.run(max_iters=iters)
    finally:
        t.close()
    return t


def _hand_loop(tree, weights, scheme, iters, arch):
    """The reference's call order written out: bin_model's optimizer and scheduler, then for k = 1, 2, ...
    update_learning_rate(k, warmup_iter) and optimize_parameters."""
    from bin_b200 import rdn
    from bin_b200.evaluate import load_weights
    from bin_b200.loss import pixel_loss
    from bin_b200.lr_scheduler import CosineAnnealingLR_Restart, MultiStepLR_Restart, warm_up
    from bin_b200.optim import Adam
    from bin_b200.trainset import DeviceBINDataset
    from test_gpu_train_driver import SEED, gts
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    random.seed(SEED)
    torch.manual_seed(SEED)
    ds = DeviceBINDataset.from_tree(tree, mode="train", device="cuda", lq_size=(3, 128, 256))
    net = rdn.bin_stage4_lstm()
    if arch:
        net.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=arch[0], D=arch[1])
    load_weights(net, weights)
    net = net.cuda().train()
    opt = Adam(net.parameters(), lr=1e-4, betas=(0.9, 0.99), weight_decay=0)
    c = {k.split(".", 1)[1]: v for k, v in SCHEMES[scheme].items()}
    if scheme == "ms":
        sched = MultiStepLR_Restart(opt, c["lr_steps"], restarts=c["restarts"], weights=c["restart_weights"],
                                    gamma=c["lr_gamma"], clear_state=c["clear_state"])
    else:
        sched = CosineAnnealingLR_Restart(opt, c["T_period"], eta_min=c["eta_min"], restarts=c["restarts"],
                                          weights=c["restart_weights"])
    step, lrs = 0, []
    while step < iters:
        for b in ds.batches(range(len(ds)), 2):
            sched.step()
            warm_up(opt, step + 1, c["warmup_iter"])
            lrs.append(opt.param_groups[0]["lr"])
            opt.zero_grad(set_to_none=True)
            outs = net(*[b["LQs"][:, k] for k in range(6)])
            loss, _ = pixel_loss(outs, gts(b), "cb", nframes=6, version=2)
            (1.0 * loss).backward()
            opt.step()
            step += 1
            if step == iters:
                break
    return net, opt, sched, lrs


def _log(save):
    path = os.path.join(save, "experiments", "bin_test", "train_bin_test.log")
    return [line.split(" - ", 1)[1] for line in open(path).read().splitlines() if "iter:" in line]


@pytest.mark.parametrize("scheme,arch", [("ms", None), ("cos", None), ("ms", (64, 6)), ("cos", (64, 6))])
def test_driver_equals_hand_loop(data, tmp_path, scheme, arch):
    """6 iterations: MultiStepLR warms up over iterations 1-2, decays at 2, restarts at 4 (weight 0.5, the Adam state
    dropped) and decays twice at 5; the cosine warms up at 1, restarts at 3 into a period of 4.  Every iteration is
    logged, and its lr: is the lr the hand loop ran that iteration with."""
    from test_gpu_train_driver import assert_same_training
    tree, weights = data
    w = weights["light" if arch else "shipped"]
    t = _driver(_options(tree, str(tmp_path), w, scheme, **{"logger.print_freq": 1}), 6, arch=arch)
    net, opt, sched, lrs = _hand_loop(tree, w, scheme, 6, arch)
    assert t.step == 6
    assert_same_training(t.net, t.opt, net, opt)
    assert t.scheduler.state_dict() == sched.state_dict()
    logged = [line.split("lr:", 1)[1].split(">", 1)[0] for line in _log(str(tmp_path))]
    assert logged == ["{:.3e}".format(v) for v in lrs]
    if scheme == "ms":
        assert float(t.opt.state[t.opt.param_groups[0]["params"][0]]["step"]) == 3.0   # restarted at iteration 4
        assert lrs[3] == 0.5e-4 and lrs[4] == 0.5e-4 * 0.25


@pytest.mark.parametrize("scheme", ["ms", "cos"])
def test_graph_equals_eager_across_restart(data, tmp_path, scheme):
    """--cuda_graph against eager over 7 iterations across the milestones and the (clear-state) restart: weights, Adam
    state, checkpoint bytes and the logged lr and losses; the graphed iterations after the first under sync-debug
    "error"."""
    from test_gpu_train_graph import _assert_same, _files
    tree, weights = data
    over = {"logger.print_freq": 1, "logger.save_checkpoint_freq": 4}
    a = _driver(_options(tree, str(tmp_path / "eager"), weights["light"], scheme, **over), 7, arch=(64, 6))
    b = _driver(_options(tree, str(tmp_path / "graph"), weights["light"], scheme, **over), 7, arch=(64, 6),
                cuda_graph=True, sync_debug="error")
    assert b._graph is not None and b.opt.capturable
    _assert_same(a.net, a.opt, b.net, b.opt)
    fa, la = _files(str(tmp_path / "eager"))
    fb, lb = _files(str(tmp_path / "graph"))
    assert sorted(fa) == sorted(fb) and len(fa) == 4
    for k in fa:
        assert fa[k] == fb[k], k
    assert la == lb and len(la) == 7


@pytest.mark.parametrize("guard", [False, True])
def test_restart_iterations_do_not_synchronise(data, tmp_path, guard):
    """Iterations 2..6, the clear-state restart at 4 included, under sync-debug "error"."""
    kw = {"max_grad_norm": 10.0, "skip_nonfinite": True} if guard else {}
    t = _driver(_options(data[0], str(tmp_path), data[1]["shipped"], "ms", **{"logger.print_freq": 3}), 6,
                sync_debug="error", **kw)
    assert t.step == 6


@pytest.mark.parametrize("scheme,at,graph", [("ms", 3, False), ("cos", 2, False), ("ms", 3, True)])
def test_resume_across_milestone_and_restart(data, tmp_path, scheme, at, graph):
    """A state saved before the restart (and, MultiStepLR, a milestone), resumed and run to 6, equals the run that
    never stopped; a state of another scheme is refused."""
    from bin_b200 import BinB200Error
    from test_gpu_train_driver import assert_same_training
    tree, weights = data
    straight = str(tmp_path / "straight")
    over = {"logger.save_checkpoint_freq": 1}
    a = _driver(_options(tree, straight, weights["light"], scheme, **over), 6, arch=(64, 6), cuda_graph=graph)
    save = str(tmp_path / "resumed")
    shutil.copytree(straight, save)
    state = os.path.join(save, "experiments", "bin_test", "training_state", f"{at}.state")
    b = _driver(_options(tree, save, None, scheme, **over, **{"path.resume_state": state}), 6, arch=(64, 6),
                cuda_graph=graph)
    assert b.step == 6
    assert_same_training(a.net, a.opt, b.net, b.opt)
    assert a.scheduler.state_dict() == b.scheduler.state_dict()
    if not graph:
        other = "cos" if scheme == "ms" else "ms"
        with pytest.raises(BinB200Error, match=r"train\.lr_scheme"):
            _driver(_options(tree, str(tmp_path / "other"), None, other, **{"path.resume_state": state}), 6,
                    arch=(64, 6))


# ----------------------------------------------------------------------------- two ranks
def _ddp_worker(rank, world, opt, port, out):
    import torch.distributed as tdist
    from bin_b200 import train as T
    os.environ["LOCAL_RANK"] = str(rank)
    torch.cuda.set_device(rank)
    tdist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        t = T.Trainer(T.parse_options(opt), deterministic=True, stdout=False, ratio=1)
        lrs = []
        orig = t.train_step

        def step(batch):
            lrs.append(t.opt.param_groups[0]["lr"])
            return orig(batch)
        t.train_step = step
        t.run(max_iters=5)
        t.close()
        flat = torch.cat([p.detach().reshape(-1) for p in t.net.parameters()])
        torch.save({"flat": flat.cpu(), "lrs": lrs, "sched": t.scheduler.state_dict()},
                   os.path.join(out, f"rank{rank}.pt"))
    finally:
        tdist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs for a world-2 NCCL run")
def test_two_ranks_step_the_same_schedule(data, tmp_path):
    import torch.multiprocessing as mp
    tree, weights = data
    opt = _options(tree, str(tmp_path), weights["shipped"], "ms", **{"datasets.train.batch_size": 4})
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_ddp_worker, args=(2, opt, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(os.path.join(str(tmp_path), f"rank{r}.pt"), weights_only=False) for r in range(2))
    assert torch.equal(r0["flat"], r1["flat"])
    assert r0["lrs"] == r1["lrs"] and len(r0["lrs"]) == 5 and r0["lrs"][3] == 0.5e-4
    assert r0["sched"] == r1["sched"]
