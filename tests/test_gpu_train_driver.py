"""The training driver (bin_b200.train) on the GPU, on a seeded PNG tree laid out as the reference's dataset script
writes it: the driver against a hand-written DeviceBINDataset -> module -> pixel_loss -> backward -> Adam loop, resume
against an uninterrupted run, the checkpoint files, the validation sums against a restated loop, ordinary iterations
under sync-debug "error", and two ranks over NCCL when two GPUs are visible.  Everything runs deterministic."""
import os
import random
import shutil
import socket

import numpy as np
import pytest
import torch

from oracle import arch_oracle as A
from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu

H, W, FIRST, NB = 352, 640, 17, 8          # 8 blurry frames per folder: 3 windows
SEED = 3


def _png(path, img):
    import cv2
    assert cv2.imwrite(path, img)


def make_tree(root, mode, folders, seed):
    """<root>/<mode>/<folder> sharp frames FIRST + 4m, <mode>_blur blurry frames FIRST + 8i, <mode>_list im_lists."""
    g = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, mode + "_list"), exist_ok=True)
    for f in folders:
        for sub in (mode, mode + "_blur"):
            os.makedirs(os.path.join(root, sub, f))
        base = g.integers(0, 256, size=(H // 8, W // 8, 3)).astype(np.float32)
        names = []
        for m in range(2 * NB - 1):
            base += g.normal(0, 3, size=base.shape).astype(np.float32)
            img = np.clip(np.kron(base, np.ones((8, 8, 1), np.float32)), 0, 255).astype(np.uint8)
            _png(os.path.join(root, mode, f, f"{FIRST + 4 * m:05d}.png"), img)
            if m % 2 == 0:
                blur = np.clip(img.astype(np.int16) + g.integers(-8, 9, size=img.shape), 0, 255).astype(np.uint8)
                names.append(f"{FIRST + 4 * m:05d}.png")
                _png(os.path.join(root, mode + "_blur", f, names[-1]), blur)
        with open(os.path.join(root, mode + "_list", f + "_im_list.txt"), "w") as fh:
            fh.write("\n".join(names))


def make_sharp_tree(root, mode, folders, seed, T=80):
    """<root>/<mode>/<folder>/00001.png ... T sharp frames, for --from_sharp (floor(T/8) - 2 = 8 blurry frames)."""
    g = np.random.default_rng(seed)
    for f in folders:
        os.makedirs(os.path.join(root, mode, f))
        base = g.integers(0, 256, size=(H // 8, W // 8, 3)).astype(np.float32)
        for k in range(1, T + 1):
            base += g.normal(0, 2, size=base.shape).astype(np.float32)
            _png(os.path.join(root, mode, f, f"{k:05d}.png"),
                 np.clip(np.kron(base, np.ones((8, 8, 1), np.float32)), 0, 255).astype(np.uint8))


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    root = tmp_path_factory.mktemp("train_tree")
    tree, sharp = str(root / "blur"), str(root / "sharp")
    make_tree(tree, "train", ["clipA", "clipB", "clipC"], 1)
    make_tree(tree, "test", ["clipV"], 2)
    make_sharp_tree(sharp, "train", ["s0", "s1"], 3)
    make_sharp_tree(sharp, "test", ["sv"], 4)
    weights = {}
    for name, sd in (("shipped", O.synth_state_dict(0)), ("light", A.synth_state_dict(0, 64, 6))):
        weights[name] = str(root / f"{name}.pth")
        torch.save(sd, weights[name])
    return {"tree": tree, "sharp": sharp, "weights": weights}


@pytest.fixture(autouse=True)
def _restore_determinism():
    yield
    torch.use_deterministic_algorithms(False)
    torch.utils.deterministic.fill_uninitialized_memory = True
    torch.cuda.set_sync_debug_mode(0)


def options(root, save, weights, **over):
    opt = {
        "name": "bin_test", "gpu_ids": [0],
        "datasets": {"train": {"name": "train", "mode": "BIN", "dataroot_LQ": root, "use_shuffle": True,
                               "n_workers": 3, "batch_size": 2, "LQ_size": [3, 128, 256]},
                     "val": {"name": "test", "mode": "BIN", "dataroot_LQ": root, "LQ_size": [3, 128, 256]}},
        "network_G": {"which_model_G": "bin_stage4", "nframes": 6, "version": 2},
        "path": {"pretrain_model_G": weights, "save_path": save, "strict_load": True, "resume_state": None},
        "train": {"lr_G": 1e-4, "lr_scheme": "ReduceLROnPlateau", "beta1": 0.9, "beta2": 0.99, "factor": 0.2,
                  "patience": 1, "epoch": 100, "pixel_criterion": "cb", "pixel_weight": 1.0, "val_freq": 1e9,
                  "manual_seed": SEED},
        "logger": {"print_freq": 2, "save_checkpoint_freq": 1e9},
    }
    for k, v in over.items():
        node = opt
        *parents, leaf = k.split(".")
        for p in parents:
            node = node[p]
        node[leaf] = v
    return opt


def driver(opt, iters, **kw):
    from bin_b200 import train as T
    t = T.Trainer(T.parse_options(opt), deterministic=True, stdout=False, **kw)
    try:
        t.run(max_iters=iters)
    finally:
        t.close()
    return t


def gts(b):
    I = {}
    for m in range(6):
        I[2 * m + 1] = b["GTenh"][:, m]
    for m in range(1, 6):
        I[2 * m] = b["GTinp"][:, m - 1]
    return [I[i] for i in (2, 4, 6, 8, 3, 5, 7, 4, 6, 5, 10, 9, 8, 7)]                  # bin_model.get_info


def sharp_dataset(root, mode, lq, rng):
    import cv2
    from bin_b200.trainset import DeviceBINDataset, DeviceClip
    clips = []
    for f in os.listdir(os.path.join(root, mode)):
        d = os.path.join(root, mode, f)
        frames = [torch.from_numpy(cv2.imread(os.path.join(d, n))) for n in sorted(os.listdir(d))]
        clips.append(DeviceClip.from_sharp(f, torch.stack(frames).cuda()))
    return DeviceBINDataset(clips, lq_size=lq, rng=rng)


def hand_loop(root, weights, iters, arch=None, checkpointing=None, from_sharp=False):
    """INTEGRATION's loop written out: seeds, dataset, net, Adam, then K steps of optimize_parameters."""
    from bin_b200 import rdn
    from bin_b200.evaluate import load_weights
    from bin_b200.loss import pixel_loss
    from bin_b200.optim import Adam
    from bin_b200.trainset import DeviceBINDataset
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    random.seed(SEED)
    torch.manual_seed(SEED)
    lq = (3, 128, 256)
    ds = sharp_dataset(root, "train", lq, random) if from_sharp else \
        DeviceBINDataset.from_tree(root, mode="train", device="cuda", lq_size=lq)
    net = rdn.bin_stage4_lstm()
    if arch:
        net.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=arch[0], D=arch[1])
    load_weights(net, weights)
    net = net.cuda().train()
    rdn.set_activation_checkpointing(net, checkpointing)
    opt = Adam(net.parameters(), lr=1e-4, betas=(0.9, 0.99), weight_decay=0)
    step = 0
    while step < iters:
        for b in ds.batches(range(len(ds)), 2):
            opt.zero_grad(set_to_none=True)
            outs = net(*[b["LQs"][:, k] for k in range(6)])
            loss, _ = pixel_loss(outs, gts(b), "cb", nframes=6, version=2)
            (1.0 * loss).backward()
            opt.step()
            step += 1
            if step == iters:
                break
    return net, opt


def assert_same_training(net_a, opt_a, net_b, opt_b):
    pa, pb = list(net_a.parameters()), list(net_b.parameters())
    assert len(pa) == len(pb)
    for a, b in zip(pa, pb):
        assert torch.equal(a, b)
    sa, sb = opt_a.state_dict(), opt_b.state_dict()
    keys = ("lr", "betas", "eps", "weight_decay", "params")
    assert [{k: g[k] for k in keys} for g in sa["param_groups"]] == [{k: g[k] for k in keys} for g in sb["param_groups"]]
    assert sorted(sa["state"]) == sorted(sb["state"])
    for k in sa["state"]:
        for n in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(sa["state"][k][n].cpu(), sb["state"][k][n].cpu()), (k, n)


# ----------------------------------------------------------------------------- 1. the driver is the hand-written loop
@pytest.mark.parametrize("variant", ["shipped", "light", "recompute", "from_sharp"])
def test_driver_equals_hand_loop(data, tmp_path, variant):
    K = 6                                                    # 9 windows, batch 2: 4 iterations per epoch
    arch = (64, 6) if variant == "light" else None
    ckpt = "recompute" if variant == "recompute" else None
    sharp = variant == "from_sharp"
    root = data["sharp"] if sharp else data["tree"]
    w = data["weights"]["light" if arch else "shipped"]
    t = driver(options(root, str(tmp_path), w), K, arch=arch, checkpointing=ckpt, from_sharp=sharp)
    if arch is None:
        assert len(list(t.net.parameters())) == 540
    net, opt = hand_loop(root, w, K, arch, ckpt, sharp)
    assert t.step == K
    assert_same_training(t.net, t.opt, net, opt)


# ----------------------------------------------------------------------------- 2, 3. resume and checkpoints
def test_resume_continues_exactly(data, tmp_path):
    from bin_b200 import rdn
    from bin_b200 import train as T
    from bin_b200.evaluate import load_weights
    straight = str(tmp_path / "straight")
    opt = options(data["tree"], straight, data["weights"]["shipped"],
                  **{"logger.save_checkpoint_freq": 2, "train.val_freq": 3})
    a = driver(opt, 7)                                      # saves 2, 4, 6 and 7; validates at 3 and 6
    na = next(a._batches())                                 # the training draws share the global `random`
    exp = os.path.join(straight, "experiments", "bin_test")
    assert sorted(os.listdir(os.path.join(exp, "models"))) == [f"{i}_G.pth" for i in (2, 4, 6, 7)]
    assert sorted(os.listdir(os.path.join(exp, "training_state"))) == [f"{i}.state" for i in (2, 4, 6, 7)]
    assert os.path.exists(os.path.join(exp, "train_bin_test.log"))
    for at in (4, 6):                                       # an epoch boundary, and inside epoch 1
        save = str(tmp_path / f"from{at}")
        shutil.copytree(straight, save)
        state = os.path.join(save, "experiments", "bin_test", "training_state", f"{at}.state")
        st = torch.load(state)
        assert set(st) == {"epoch", "iter", "schedulers", "optimizers"} and st["iter"] == at
        b = driver(options(data["tree"], save, None, **{"logger.save_checkpoint_freq": 2, "train.val_freq": 3,
                                                          "path.resume_state": state}), 7)
        assert b.step == 7
        assert_same_training(a.net, a.opt, b.net, b.opt)
        assert a.scheduler.state_dict() == b.scheduler.state_dict()
        nb = next(b._batches())
        assert na["key"] == nb["key"] and torch.equal(na["LQs"], nb["LQs"])

    # 3. the checkpoint: 1 332 keys, strict into bin_stage4_lstm, the trained net's window, evaluate's prefixes
    path = os.path.join(exp, "models", "7_G.pth")
    sd = torch.load(path)
    assert len(sd) == 1332 and all(v.device.type == "cpu" for v in sd.values())
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(sd, strict=True)
    net = net.cuda().eval()
    fr = [f.cuda() for f in O.synth_frames(6, 1, 64, 96, seed=9)]
    with torch.no_grad():
        for x, y in zip(net(*fr), a.net(*fr)):
            assert torch.equal(x, y)
    prefixed = str(tmp_path / "prefixed.pth")
    torch.save({"InterpNet." + k: v for k, v in sd.items()}, prefixed)
    other = rdn.bin_stage4_lstm()
    load_weights(other, prefixed)
    assert all(torch.equal(x, y) for x, y in zip(other.state_dict().values(), sd.values()))
    assert T.resume_position(st["epoch"], st["iter"], a.iters_per_epoch) == divmod(6, 4)


# ----------------------------------------------------------------------------- 4. validation
def test_validation_sums_equal_restated_loop(data, tmp_path):
    from bin_b200.loss import pixel_loss
    from bin_b200.metrics import calculate_psnr, calculate_ssim
    from bin_b200.streaming import tensor2img_u8
    from bin_b200.trainset import DeviceBINDataset
    t = driver(options(data["tree"], str(tmp_path), data["weights"]["shipped"]), 2)
    log = t.validate()
    got = list(t.val_sums)
    assert t.validate() == log and t.val_sums == got        # every validation scores the same crops
    vs = DeviceBINDataset.from_tree(data["tree"], mode="test", lq_size=(3, 128, 256), rng=random.Random(SEED))
    vs.rng = random.Random(SEED)
    sums = [0] * 43
    with torch.no_grad():
        for i in range(len(vs)):
            b = vs.batch([i])
            outs = t.net(*[b["LQs"][:, k] for k in range(6)])
            loss, lst = pixel_loss(outs, gts(b), "cb", nframes=6, version=2)
            terms = [x.item() for x in lst] + [loss.item()]
            for k, g in enumerate(gts(b)):
                a, r = tensor2img_u8(outs[k][0]), tensor2img_u8(g[0])
                terms.append(calculate_psnr(a, r))
            for k, g in enumerate(gts(b)):
                terms.append(calculate_ssim(tensor2img_u8(outs[k][0]), tensor2img_u8(g[0])))
            for k, v in enumerate(terms):
                sums[k] += v
    assert got == [float(v) for v in sums] + [float(len(vs))]
    assert log[4] == sums[14] / len(vs)


# ----------------------------------------------------------------------------- 5. no host synchronisation
@pytest.mark.parametrize("guard", [False, True])
def test_ordinary_iterations_do_not_synchronise(data, tmp_path, guard):
    kw = {"max_grad_norm": 10.0, "skip_nonfinite": True} if guard else {}
    opt = options(data["tree"], str(tmp_path), data["weights"]["shipped"], **{"logger.print_freq": 3})
    t = driver(opt, 6, sync_debug="error", **kw)             # iterations 2..6 under "error", across an epoch boundary
    assert t.step == 6


# ----------------------------------------------------------------------------- the command line
def test_command_line_trains_and_evaluate_loads(data, tmp_path):
    import subprocess
    import sys
    import yaml
    opt = options(data["tree"], str(tmp_path), data["weights"]["shipped"],
                  **{"train.epoch": 1, "train.val_freq": 2, "logger.print_freq": 1})
    yml = str(tmp_path / "train.yml")
    with open(yml, "w") as fh:
        yaml.safe_dump(opt, fh)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "bin_b200.train", "-opt", yml, "--deterministic"], cwd=root,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "# Validation #" in r.stdout and "gpu_ids is ignored" in r.stdout
    log = open(os.path.join(str(tmp_path), "experiments", "bin_test", "train_bin_test.log")).read()
    assert "<epoch:  0, iter:       4, lr:1.000e-04>" in log
    from bin_b200 import rdn
    from bin_b200.evaluate import load_weights
    load_weights(rdn.bin_stage4_lstm(), os.path.join(str(tmp_path), "experiments", "bin_test", "models", "4_G.pth"))


# ----------------------------------------------------------------------------- 6. two ranks
def _ddp_worker(rank, world, opt, port, out):
    import torch.distributed as tdist
    from bin_b200 import train as T
    os.environ["LOCAL_RANK"] = str(rank)
    torch.cuda.set_device(rank)
    tdist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        t = T.Trainer(T.parse_options(opt), deterministic=True, stdout=False, ratio=1)
        losses = []
        orig = t.train_step

        def step(batch):
            loss, lst = orig(batch)
            losses.append(loss.detach().clone())
            return loss, lst
        t.train_step = step
        t.run(max_iters=2)
        t.close()
        flat = torch.cat([p.detach().reshape(-1) for p in t.net.parameters()])
        torch.save({"flat": flat.cpu(), "loss": torch.stack(losses).cpu()}, os.path.join(out, f"rank{rank}.pt"))
    finally:
        tdist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs for a world-2 NCCL run")
def test_two_ranks_agree(data, tmp_path):
    import torch.multiprocessing as mp
    from bin_b200 import rdn
    from bin_b200 import train as T
    from bin_b200.evaluate import load_weights
    from bin_b200.loss import pixel_loss
    from bin_b200.optim import Adam
    from bin_b200.trainset import DeviceBINDataset
    opt = options(data["tree"], str(tmp_path), data["weights"]["shipped"], **{"datasets.train.batch_size": 4})
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_ddp_worker, args=(2, opt, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(os.path.join(str(tmp_path), f"rank{r}.pt")) for r in range(2))
    assert torch.equal(r0["flat"], r1["flat"])
    # one process: the same per-rank batches, DDP's gradient (the mean over ranks) by hand
    torch.use_deterministic_algorithms(True)
    sets = []
    for r in range(2):
        ds = DeviceBINDataset.from_tree(data["tree"], mode="train", lq_size=(3, 128, 256), rng=random.Random(SEED))
        sampler = T.DistIterSampler(len(ds), 2, r, 1)
        sampler.set_epoch(0)
        sets.append(ds.batches(iter(sampler), 2))
    net = rdn.bin_stage4_lstm()
    load_weights(net, data["weights"]["shipped"])
    net = net.cuda().train()
    params = list(net.parameters())
    adam = Adam(params, lr=1e-4, betas=(0.9, 0.99))
    losses = []
    for _ in range(2):
        grads, ls = [], []
        for it in sets:
            b = next(it)
            adam.zero_grad(set_to_none=True)
            loss, _ = pixel_loss(net(*[b["LQs"][:, k] for k in range(6)]), gts(b), "cb", nframes=6, version=2)
            loss.backward()
            grads.append([p.grad.clone() for p in params])
            ls.append(loss.detach())
        for p, g0, g1 in zip(params, *grads):
            p.grad = (g0 + g1) / 2
        adam.step()
        losses.append(torch.stack(ls))
    want = torch.stack(losses).cpu()
    got = torch.stack([r0["loss"], r1["loss"]], 1)
    rel = ((got - want).abs() / want.abs()).max().item()
    print(f"two ranks vs one process: max relative loss difference {rel:.3e} (bar 1e-4: the ranks' gradients are "
          "summed in another order by the all-reduce)")
    assert rel <= 1e-4
