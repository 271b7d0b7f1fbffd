"""The training step captured in a CUDA graph (DESIGN.md §4p): the device-scalar Adam against the host's bias
corrections over 100 000 steps, Adam(capturable=True) against its own default and torch's capturable Adam, replays
against eager steps bit for bit (both windows, both checkpointing modes, a frozen backbone, a learning-rate change, the
guard), weights re-packed on every replay, and Trainer(cuda_graph=True) against the eager driver.  Everything runs
under torch.use_deterministic_algorithms(True)."""
import copy
import math
import os

import numpy as np
import pytest
import torch

from oracle import arch_oracle as A
from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu

B, H, W = 2, 64, 128
K = 5                                                       # steps compared


@pytest.fixture(autouse=True)
def _deterministic():
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    yield
    torch.use_deterministic_algorithms(False)
    torch.utils.deterministic.fill_uninitialized_memory = True
    torch.cuda.set_sync_debug_mode(0)


# ----------------------------------------------------------------------------- 1. the device's bias corrections
@pytest.mark.parametrize("betas", [(0.9, 0.99), (0.9, 0.999)])
def test_device_scalars_equal_host_bias_corrections(betas):
    """lr / bc1 and 1 / sqrt(bc2) as adam_scalars_kernel forms them, for steps 1..100 000, against what
    Adam._launch passes (1 - beta ** step in Python doubles, as fp32) and launch_adam_step forms from it."""
    from bin_b200._lib import check, lib
    from bin_b200.optim import SCALARS_DTYPE, Adam
    N, lr = 100_000, 1e-4
    p = torch.nn.Parameter(torch.zeros(4, device="cuda"))
    p.grad = torch.zeros(4, device="cuda")
    opt = Adam([p], lr=lr, betas=betas, capturable=True)
    opt.step()                                              # builds the table and the scalar block
    tab = opt._tables[(0, 0)]
    blk = np.zeros(1, dtype=SCALARS_DTYPE)
    blk["beta1"], blk["beta2"], blk["lr"] = betas[0], betas[1], lr
    blk["audit"] = opt._audit_bufs[0].data_ptr()            # the record an unguarded step reads: never skip, coef 1
    tab.sc.copy_(torch.from_numpy(blk.view(np.float32).copy()))
    got = torch.empty((N, 2), device="cuda")
    args = (tab.dev.data_ptr(), tab.prefix.data_ptr(), tab.n, tab.nchunks, 0.0, betas[0], betas[1], 1e-8, 0.0, 1.0, 1.0,
            1.0, tab.sc.data_ptr(), torch.cuda.current_stream().cuda_stream)
    for i in range(N):
        check(lib().bin_adam_step(*args))
        got[i].copy_(tab.sc[10:12])
    got = got.cpu().numpy()
    want = np.empty((N, 2), dtype=np.float32)
    lr32 = np.float32(lr)
    for i in range(N):
        step = float(i) + 1.0
        bc1, bc2 = np.float32(1.0 - betas[0] ** step), np.float32(1.0 - betas[1] ** step)
        want[i, 0] = lr32 / bc1
        want[i, 1] = np.float32(1.0) / np.sqrt(bc2)
    bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))
    assert bad[0].size == 0, [(int(r) + 1, int(c)) for r, c in zip(*bad)][:10]
    assert float(tab.sc[9]) == N                            # the count the block restarted from, advanced N times


# ----------------------------------------------------------------------------- 2. capturable Adam on random tensors
SHAPES = [(96, 64, 3, 3), (96,), (5000,), (3, 7), (4096 * 3 + 5,)]


def _params(seed):
    """Weights of the size of the window's (|w| < 0.5), where the existing Adam test's 2e-7 bar against torch is ~1 ulp."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(s, device="cuda", generator=g) * 0.1) for s in SHAPES]


def _grads(ps, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(p.shape, device="cuda", generator=g) * 1e-2 for p in ps]


def test_capturable_adam_equals_default_and_torch():
    from bin_b200.optim import Adam
    hyper = dict(lr=1e-4, betas=(0.9, 0.99), weight_decay=1e-5)
    pa, pb, pc = _params(1), _params(1), _params(1)
    ours, plain = Adam(pa, capturable=True, **hyper), Adam(pb, **hyper)
    ref = torch.optim.Adam(pc, capturable=True, foreach=False, **hyper)
    for step in range(4):
        if step == 2:                                       # a scheduler's write
            for o in (ours, plain, ref):
                o.param_groups[0]["lr"] = 5e-5
        gs = _grads(pa, 10 + step)
        for ps in (pa, pb, pc):
            for p, g in zip(ps, gs):
                if p.grad is None:
                    p.grad = g.clone()
                else:
                    p.grad.copy_(g)                         # capturable: the same gradient tensors every step
        ours.step()
        plain.step()
        ref.step()
    for a, b in zip(pa, pb):
        assert torch.equal(a, b)
    for a, b in zip(pa, pb):
        sa, sb = ours.state[a], plain.state[b]
        assert sa["step"].is_cuda and float(sa["step"]) == float(sb["step"]) == 4.0
        assert torch.equal(sa["exp_avg"], sb["exp_avg"]) and torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"])
    worst = max(float((a.detach() - c.detach()).abs().max()) for a, c in zip(pa, pc))
    assert worst <= 2e-7, worst
    # state dicts: CPU steps, the default optimizer's bytes; into torch's capturable Adam and back, and across modes
    sd, sdp = ours.state_dict(), plain.state_dict()
    assert all(not st["step"].is_cuda for st in sd["state"].values())
    assert sd["param_groups"] == sdp["param_groups"]
    back = Adam(_params(2), capturable=True, **hyper)
    torch_back = torch.optim.Adam(_params(2), capturable=True, **hyper)
    torch_back.load_state_dict(copy.deepcopy(sd))
    back.load_state_dict(copy.deepcopy(torch_back.state_dict()))
    to_plain = Adam(_params(2), **hyper)
    to_plain.load_state_dict(copy.deepcopy(back.state_dict()))
    from_plain = Adam(_params(2), capturable=True, **hyper)
    from_plain.load_state_dict(copy.deepcopy(sdp))
    for o in (back, to_plain, from_plain):
        osd = o.state_dict()
        for k in sd["state"]:
            for n in ("step", "exp_avg", "exp_avg_sq"):
                assert torch.equal(osd["state"][k][n].cpu(), sd["state"][k][n].cpu()), (o, k, n)
    # a resumed capturable optimizer steps as the default one does
    qa, qb = _params(1), _params(1)
    for q, a in zip(qa + qb, pa + pa):
        q.data.copy_(a.data)
    oa, ob = Adam(qa, capturable=True, **hyper), Adam(qb, **hyper)
    oa.load_state_dict(copy.deepcopy(sdp))
    ob.load_state_dict(copy.deepcopy(sd))
    gs = _grads(qa, 30)
    for q, r, g in zip(qa, qb, gs):
        q.grad, r.grad = g.clone(), g.clone()
    oa.step()
    ob.step()
    assert all(torch.equal(a, b) for a, b in zip(qa, qb))


def test_capturable_refusals():
    from bin_b200 import BinB200Error
    from bin_b200.optim import Adam
    p = torch.nn.Parameter(torch.zeros(8, device="cuda"))
    with pytest.raises(ValueError, match="capturable"):
        Adam([p], skip_nonfinite=True, loss_scale_backoff=True, capturable=True)
    opt = Adam([p, torch.nn.Parameter(torch.zeros(3, device="cuda"))], capturable=True)
    p.grad = torch.zeros(8, device="cuda")
    with pytest.raises(BinB200Error, match="gradient"):
        opt.step()                                          # the second parameter has none


# ----------------------------------------------------------------------------- 3-6. replays against eager steps
def _net(arch, ckpt, frozen):
    from bin_b200 import rdn
    net = rdn.bin_stage4_lstm()
    if arch:
        net.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=64, D=6)
        net.load_state_dict(A.synth_state_dict(0, 64, 6))
    else:
        net.load_state_dict(O.synth_state_dict(0))
    net = net.cuda().train()
    rdn.set_activation_checkpointing(net, ckpt)
    if frozen:
        for p in net.model.model1_1.parameters():
            p.requires_grad_(False)
    return net, [p for p in net.parameters() if p.requires_grad]


def _batches(n, bad=None):
    """n seeded (17, B, 3, H, W) buffers on the device; batch `bad` holds an inf in its first frame."""
    g = torch.Generator(device="cuda").manual_seed(7)
    out = [torch.rand((17, B, 3, H, W), device="cuda", generator=g) for _ in range(n)]
    if bad is not None:
        out[bad][0, 0, 1, 5, 9] = math.inf
    return out


def _step(net, opt, buf, set_to_none):
    from bin_b200.loss import pixel_loss
    from bin_b200.train import gt_list
    opt.zero_grad(set_to_none=set_to_none)
    b = {"LQs": buf[0:6].transpose(0, 1), "GTenh": buf[6:12].transpose(0, 1), "GTinp": buf[12:].transpose(0, 1)}
    outs = net(*[b["LQs"][:, k] for k in range(6)])
    loss, _ = pixel_loss(outs, gt_list(b), "cb", nframes=6, version=2)
    loss.backward()
    opt.step()
    return loss, outs


def _lr_change(opt, k, at):
    if k == at:
        for grp in opt.param_groups:
            grp["lr"] = grp["lr"] * 0.2                     # ReduceLROnPlateau's write


def _eager(arch, ckpt, frozen, batches, lr_at=None, **guard):
    from bin_b200.optim import Adam
    net, ps = _net(arch, ckpt, frozen)
    opt = Adam(ps, lr=1e-4, betas=(0.9, 0.99), **guard)
    losses = []
    for k, buf in enumerate(batches):
        _lr_change(opt, k, lr_at)
        loss, _ = _step(net, opt, buf, True)
        losses.append(loss.detach().clone())
    opt.resolve()
    return net, opt, losses


class _Graphed:
    """Warm-up step eagerly on a side stream, then one capture on a static batch, then replays."""

    def __init__(self, arch, ckpt, frozen, first, **guard):
        from bin_b200 import rdn
        from bin_b200.optim import Adam
        self.net, ps = _net(arch, ckpt, frozen)
        self.opt = Adam(ps, lr=1e-4, betas=(0.9, 0.99), capturable=True, **guard)
        self.static = first.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            loss, _ = _step(self.net, self.opt, self.static, True)
            self.losses = [loss.detach().clone()]
            rdn.take_workspace(self.static.device)
        torch.cuda.current_stream().wait_stream(side)
        self.graph, self.capture = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        with torch.cuda.graph(self.graph, stream=self.capture):
            self.loss, self.outs = _step(self.net, self.opt, self.static, False)
            self.ws = rdn.take_workspace(self.static.device)

    def run(self, buf):
        self.static.copy_(buf)
        self.opt.replay(self.graph)
        self.losses.append(self.loss.detach().clone())


def _graphed(arch, ckpt, frozen, batches, lr_at=None, **guard):
    g = _Graphed(arch, ckpt, frozen, batches[0], **guard)
    for k, buf in enumerate(batches[1:], 1):
        _lr_change(g.opt, k, lr_at)
        g.run(buf)
    g.opt.resolve()
    return g


def _assert_same(net_a, opt_a, net_b, opt_b):
    for (na, a), (nb, b) in zip(net_a.named_parameters(), net_b.named_parameters()):
        assert na == nb and torch.equal(a, b), na
    sa, sb = opt_a.state_dict(), opt_b.state_dict()
    assert sa["param_groups"] == sb["param_groups"]
    assert sorted(sa["state"]) == sorted(sb["state"]) and len(sa["state"]) > 0
    for k in sa["state"]:
        for n in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(sa["state"][k][n].cpu(), sb["state"][k][n].cpu()), (k, n)


@pytest.mark.parametrize("arch,ckpt,frozen", [(None, None, False), (None, "recompute", False), ("light", None, False),
                                              ("light", "recompute", False), ("light", None, True)])
def test_replays_equal_eager_steps(arch, ckpt, frozen):
    batches = _batches(K)
    net_e, opt_e, loss_e = _eager(arch, ckpt, frozen, batches)
    g = _graphed(arch, ckpt, frozen, batches)
    if arch is None and not frozen:
        assert len(list(g.net.parameters())) == 540
    assert [float(x) for x in g.losses] == [float(x) for x in loss_e]
    _assert_same(net_e, opt_e, g.net, g.opt)


def test_learning_rate_change_between_replays():
    batches = _batches(K)
    net_e, opt_e, loss_e = _eager("light", None, False, batches, lr_at=3)
    g = _graphed("light", None, False, batches, lr_at=3)
    assert [float(x) for x in g.losses] == [float(x) for x in loss_e]
    assert g.opt.param_groups[0]["lr"] == opt_e.param_groups[0]["lr"] == 1e-4 * 0.2
    _assert_same(net_e, opt_e, g.net, g.opt)


@pytest.mark.parametrize("guard", [dict(skip_nonfinite=True), dict(skip_nonfinite=True, max_grad_norm=1e-3)])
def test_guard_skips_a_replay(guard):
    bad = 2
    batches = _batches(K, bad=bad)
    net_e, opt_e, _ = _eager("light", None, False, batches, **guard)
    g = _Graphed("light", None, False, batches[0], **guard)
    for k, buf in enumerate(batches[1:], 1):
        if k == bad:
            before = [p.detach().clone() for p in g.net.parameters()]
            state = {n: [g.opt.state[p][n].clone() for p in g.opt.param_groups[0]["params"]]
                     for n in ("step", "exp_avg", "exp_avg_sq")}
        g.run(buf)
        if k == bad:
            assert all(torch.equal(a, b) for a, b in zip(before, g.net.parameters()))
            for n, ts in state.items():
                assert all(torch.equal(a, g.opt.state[p][n]) for a, p in zip(ts, g.opt.param_groups[0]["params"])), n
            g.opt.resolve()
            assert g.opt.skipped_steps == 1 and g.opt.last_nonfinite_param is not None
    g.opt.resolve()
    assert g.opt.skipped_steps == opt_e.skipped_steps == 1
    assert g.opt.last_grad_norm == opt_e.last_grad_norm
    _assert_same(net_e, opt_e, g.net, g.opt)


def test_weights_are_repacked_every_replay():
    """After 3 replays an eager forward from freshly packed weights equals the forward of the next replay."""
    batches = _batches(5)
    g = _Graphed("light", None, False, batches[0])
    for buf in batches[1:4]:
        g.run(buf)
    for m in (g.net.model.model1_1, g.net.model.model2_1, g.net.model.model3_1, g.net.model.model4_1):
        for slot in [k for k in m.__dict__ if k.startswith("_pack_")]:
            del m.__dict__[slot]
    g.static.copy_(batches[4])
    b = g.static[0:6].transpose(0, 1)
    eager = [o.detach().clone() for o in g.net(*[b[:, k] for k in range(6)])]
    g.opt.replay(g.graph)
    for x, y in zip(eager, g.outs):
        assert torch.equal(x, y)


# ----------------------------------------------------------------------------- 7. the driver
def _driver(root, save, weights, iters, **kw):
    from bin_b200 import train as T
    from test_gpu_train_driver import options
    opt = options(root, save, weights, **{"logger.save_checkpoint_freq": 3, "train.val_freq": 3,
                                          "logger.print_freq": 2})
    t = T.Trainer(T.parse_options(opt), deterministic=True, stdout=False, **kw)
    try:
        t.run(max_iters=iters)
    finally:
        t.close()
    return t


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    from test_gpu_train_driver import make_tree
    root = tmp_path_factory.mktemp("graph_tree")
    tree = str(root / "blur")
    make_tree(tree, "train", ["clipA", "clipB", "clipC"], 1)
    make_tree(tree, "test", ["clipV"], 2)
    w = str(root / "shipped.pth")
    torch.save(O.synth_state_dict(0), w)
    return tree, w


def _files(save):
    exp = os.path.join(save, "experiments", "bin_test")
    out = {}
    for sub in ("models", "training_state"):
        for n in sorted(os.listdir(os.path.join(exp, sub))):
            out[os.path.join(sub, n)] = open(os.path.join(exp, sub, n), "rb").read()
    log = open(os.path.join(exp, "train_bin_test.log")).read().splitlines()
    return out, [line.split(" - ", 1)[1] for line in log if "iter:" in line]


def test_driver_graph_equals_eager(data, tmp_path):
    """7 iterations (a validation and a ReduceLROnPlateau step at 3 and 6, checkpoints at 3, 6 and 7, losses logged
    every 2), the graphed ones under sync-debug "error"; then a resume of the graphed run from iteration 3."""
    tree, w = data
    a = _driver(tree, str(tmp_path / "eager"), w, 7)
    b = _driver(tree, str(tmp_path / "graph"), w, 7, cuda_graph=True, sync_debug="error")
    assert b.cuda_graph and b._graph is not None and not a.cuda_graph
    _assert_same(a.net, a.opt, b.net, b.opt)
    fa, la = _files(str(tmp_path / "eager"))
    fb, lb = _files(str(tmp_path / "graph"))
    assert sorted(fa) == sorted(fb) and len(fa) == 6
    for k in fa:
        assert fa[k] == fb[k], k
    assert la == lb and any("Validation" in line for line in la)
    # resume the graphed run's checkpoint at 3, graphed
    import shutil
    save = str(tmp_path / "resumed")
    shutil.copytree(str(tmp_path / "graph"), save)
    state = os.path.join(save, "experiments", "bin_test", "training_state", "3.state")
    from bin_b200 import train as T
    from test_gpu_train_driver import options
    opt = options(tree, save, None, **{"logger.save_checkpoint_freq": 3, "train.val_freq": 3, "logger.print_freq": 2,
                                        "path.resume_state": state})
    c = T.Trainer(T.parse_options(opt), deterministic=True, stdout=False, cuda_graph=True)
    try:
        c.run(max_iters=7)
    finally:
        c.close()
    _assert_same(a.net, a.opt, c.net, c.opt)


def test_driver_honours_graph_switch(data, tmp_path, monkeypatch):
    tree, w = data
    monkeypatch.setenv("BIN_B200_GRAPH", "0")
    t = _driver(tree, str(tmp_path), w, 2, cuda_graph=True)
    assert not t.cuda_graph and t._graph is None and not t.opt.capturable


def test_command_line_flag(data, tmp_path):
    import subprocess
    import sys
    import yaml
    from test_gpu_train_driver import options
    tree, w = data
    opt = options(tree, str(tmp_path), w, **{"train.epoch": 1, "train.val_freq": 1e9, "logger.print_freq": 2})
    yml = str(tmp_path / "train.yml")
    with open(yml, "w") as fh:
        yaml.safe_dump(opt, fh)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "bin_b200.train", "-opt", yml, "--deterministic", "--cuda_graph"],
                       cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "iter:       4" in r.stdout
