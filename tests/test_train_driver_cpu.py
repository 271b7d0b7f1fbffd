"""The training driver's host logic (bin_b200.train): option parsing, the samplers against a restatement of
data/data_sampler.py DistIterSampler, the print / val / save / epoch schedule, the resume position, ReduceLROnPlateau
on stubbed validation losses, the log messages, and the validation-sum all-reduce under gloo with 2 processes."""
import copy
import math
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from bin_b200 import BinB200Error
from bin_b200 import train as T

YML = {                                     # options/train/train_adobe_stage4.yml, as yaml.safe_load reads it
    "name": "adobe_stage4", "use_tb_logger": True, "model": "bin", "distortion": "blur", "scale": 4, "gpu_ids": [2, 3],
    "datasets": {
        "train": {"name": "train", "mode": "BIN", "random_reverse": False, "border_mode": False,
                  "dataroot_GT": "/d/Adobe_240fps_blur", "dataroot_LQ": "/d/Adobe_240fps_blur", "use_shuffle": True,
                  "n_workers": 3, "batch_size": 2, "LQ_size": [3, 128, 256], "use_flip": True, "use_rot": True,
                  "color": "RGB"},
        "val": {"name": "test", "mode": "BIN", "task": "deblur_interp", "dataroot_GT": "/d/Adobe_240fps_blur/",
                "dataroot_LQ": "/d/Adobe_240fps_blur/", "LQ_size": [3, 128, 256], "cache_data": False,
                "padding": "new_info", "save_path": "/d/Results"}},
    "network_G": {"which_model_G": "bin_stage4", "nframes": 6, "version": 2},
    "path": {"pretrain_model_G": "./model_weights/adobe_bin.pth", "save_path": "/d/", "strict_load": True,
             "resume_state": None},
    "train": {"input_frames": 6, "lr_G": 1e-4, "lr_scheme": "ReduceLROnPlateau", "beta1": 0.9, "beta2": 0.99,
              "factor": 0.2, "patience": 1, "epoch": 100, "pixel_criterion": "cb", "pixel_weight": 1.0,
              "ssim_weight": 0.01, "val_freq": 1e4, "manual_seed": 0},
    "logger": {"print_freq": 100, "save_checkpoint_freq": 5000.0},
}


def with_(**over):
    opt = copy.deepcopy(YML)
    for k, v in over.items():
        node = opt
        *parents, leaf = k.split(".")
        for p in parents:
            node = node[p]
        if v is None:
            node.pop(leaf, None)
        else:
            node[leaf] = v
    return opt


def test_every_honoured_key():
    o = T.parse_options(YML)
    assert (o.name, o.train_root, o.train_mode, o.batch_size, o.train_lq_size, o.use_shuffle) == \
        ("adobe_stage4", "/d/Adobe_240fps_blur", "train", 2, (3, 128, 256), True)
    assert (o.val_root, o.val_mode, o.val_lq_size) == ("/d/Adobe_240fps_blur/", "test", (3, 128, 256))
    assert o.version == 2
    assert (o.pretrain_model_G, o.strict_load, o.resume_state, o.save_path) == \
        ("./model_weights/adobe_bin.pth", True, None, "/d/")
    assert (o.lr, o.beta1, o.beta2, o.weight_decay, o.pixel_criterion, o.pixel_weight) == (1e-4, 0.9, 0.99, 0.0, "cb", 1.0)
    assert (o.factor, o.patience, o.epochs, o.val_freq, o.manual_seed) == (0.2, 1, 100, 10000, 0)
    assert (o.print_freq, o.save_freq) == (100, 5000)
    assert o.ignored == ["gpu_ids", "datasets.train.n_workers"]
    assert o.experiments_root == "/d/experiments/adobe_stage4"
    assert o.models_dir == "/d/experiments/adobe_stage4/models"
    assert o.state_dir == "/d/experiments/adobe_stage4/training_state"
    o = T.parse_options(with_(**{"train.weight_decay_G": 1e-5, "path.strict_load": False, "path.resume_state": "~/r",
                                 "datasets.val": None, "train.pixel_criterion": "l2", "network_G.version": 1}))
    assert (o.weight_decay, o.strict_load, o.val_root, o.pixel_criterion, o.version) == (1e-5, False, None, "l2", 1)
    assert o.resume_state == os.path.expanduser("~/r")


@pytest.mark.parametrize("key,value", [
    ("train.lr_scheme", "MultiStepLR"), ("train.lr_scheme", "CosineAnnealingLR_Restart"),
    ("train.ft_tsa_only", 50000), ("network_G.which_model_G", "bin_stage3"), ("network_G.nframes", 4),
    ("train.pixel_criterion", "ssim")])
def test_rejected_keys_name_the_key(key, value):
    with pytest.raises(BinB200Error, match=key.replace(".", r"\.")):
        T.parse_options(with_(**{key: value}))


def test_missing_key_is_named():
    with pytest.raises(BinB200Error, match=r"train\.lr_G is missing"):
        T.parse_options(with_(**{"train.lr_G": None}))


class RefDistIterSampler:
    """data/data_sampler.py DistIterSampler, restated."""

    def __init__(self, n, num_replicas, rank, ratio=100):
        self.n, self.num_replicas, self.rank, self.epoch = n, num_replicas, rank, 0
        self.num_samples = int(math.ceil(n * ratio / num_replicas))
        self.total_size = self.num_samples * num_replicas

    def __iter__(self):
        g = torch.Generator()
        g.manual_seed(self.epoch)
        indices = torch.randperm(self.total_size, generator=g).tolist()
        indices = [v % self.n for v in indices]
        indices = indices[self.rank:self.total_size:self.num_replicas]
        assert len(indices) == self.num_samples
        return iter(indices)


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("n,ratio", [(1, 1), (9, 1), (10, 3), (37, 100)])
def test_sampler_matches_dist_iter_sampler(world, n, ratio):
    for rank in range(world):
        s, ref = T.DistIterSampler(n, world, rank, ratio), RefDistIterSampler(n, world, rank, ratio)
        assert len(s) == ref.num_samples
        for epoch in (0, 1, 7):
            s.set_epoch(epoch)
            ref.epoch = epoch
            assert list(s) == list(ref)
    m = T.make_sampler(n, world, 0, ratio)
    if world == 1:                                          # create_dataloader: shuffle=False, no sampler
        assert isinstance(m, T.SequentialSampler) and list(m) == list(range(n)) and len(m) == n
    else:
        assert isinstance(m, T.DistIterSampler)


def test_per_rank_batch():
    assert [T.per_rank_batch(8, w) for w in (1, 2, 4, 8)] == [8, 4, 2, 1]
    with pytest.raises(BinB200Error, match="not divisible"):
        T.per_rank_batch(6, 4)


def test_schedule():
    ev = {s: T.events(s, print_freq=2, val_freq=3, save_freq=6) for s in range(1, 13)}
    assert [s for s in ev if "print" in ev[s]] == [2, 4, 6, 8, 10, 12]
    assert [s for s in ev if "val" in ev[s]] == [3, 6, 9, 12]
    assert [s for s in ev if "save" in ev[s]] == [6, 12]
    assert ev[6] == ("print", "val", "save") and ev[1] == ()
    assert T.events(10, 0, 0, 0) == ()
    # epochs: iteration s runs in epoch (s - 1) // ipe
    ipe = 4
    assert [T.resume_position((s - 1) // ipe if s else 0, s, ipe) for s in range(0, 10)] == \
        [(0, 0), (0, 1), (0, 2), (0, 3), (1, 0), (1, 1), (1, 2), (1, 3), (2, 0), (2, 1)]


def test_resume_position_checks_the_epoch():
    assert T.resume_position(2, 12, 4) == (3, 0)            # saved after the last batch of epoch 2
    assert T.resume_position(3, 13, 4) == (3, 1)
    with pytest.raises(BinB200Error, match="state says epoch 1"):
        T.resume_position(1, 13, 4)                          # another batch size or dataset than the saved run's
    with pytest.raises(BinB200Error):
        T.resume_position(0, 3, 0)


def test_plateau_steps_on_stubbed_validation_losses():
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=1e-4)
    s = torch.optim.lr_scheduler.ReduceLROnPlateau(opt, "min", factor=0.2, patience=1)
    lrs = []
    for v in (1.0, 0.9, 0.95, 0.96, 0.97, 0.5, 0.6, 0.7):
        s.step(v)
        lrs.append(opt.param_groups[0]["lr"])
    assert lrs == pytest.approx([1e-4, 1e-4, 1e-4, 2e-5, 2e-5, 2e-5, 2e-5, 4e-6])
    sd = s.state_dict()                                     # what <iter>.state carries
    s2 = torch.optim.lr_scheduler.ReduceLROnPlateau(torch.optim.SGD([p], lr=1.0), "min", factor=0.2, patience=1)
    s2.load_state_dict(sd)
    assert s2.best == 0.5 and s2.num_bad_epochs == sd["num_bad_epochs"]


def test_gt_list_is_get_info():
    b = {"GTenh": torch.arange(6).view(1, 6), "GTinp": 10 + torch.arange(5).view(1, 5)}
    # I1, I3, .. I11 = GTenh[:, 0..5]; I2, I4, .. I10 = GTinp[:, 0..4] (feed_data)
    I = {2 * m + 1: m for m in range(6)} | {2 * m: 10 + m - 1 for m in range(1, 6)}
    want = [I[i] for i in (2, 4, 6, 8, 3, 5, 7, 4, 6, 5, 10, 9, 8, 7)]
    assert [int(t) for t in T.gt_list(b)] == want


def test_messages():
    avg = [0.01 * (i + 1) for i in range(14)] + [0.5]
    m = T.train_message(3, 12345, 1e-4, avg, None)
    assert m.startswith("<epoch:  3, iter:  12,345, lr:1.000e-04> 0: 1.0000e-02 1: 2.0000e-02 ")
    assert m.endswith("13: 1.4000e-01 Al: 5.0000e-01")
    g = T.train_message(0, 1, 2e-5, avg, (2, 3.5))
    assert g.endswith("Al: 5.0000e-01 skipped: 2 grad_norm: 3.5000e+00")
    assert T.train_message(0, 1, 2e-5, avg, (0, None)).endswith("grad_norm: n/a")
    sums = [2.0 * (i + 1) for i in range(14)] + [3.0] + [60.0 + i for i in range(14)] + [1.5] * 14 + [2.0]
    log = T.val_log(sums)
    avg_log, avg_psnr, psnr, ssim, loss = log
    assert list(avg_log) == [f"Al{i}" for i in range(14)] + ["Al"]
    assert list(avg_psnr) == [f"Ap{i}" for i in range(14)] + ["Ap"]
    assert avg_log["Al0"] == 1.0 and avg_log["Al"] == 1.5 and loss == 1.5
    assert avg_psnr["Ap13"] == 36.5 and psnr == sum((60.0 + i) / 2 for i in range(14)) / 14 and ssim == 0.75
    v = T.val_message(1, 2000, log)
    assert v.startswith("<epoch:  1, iter:   2,000> # Validation # Al0: 1.0000e+00 ")
    assert "Al: 1.5000e+00 Ap0: 30.0000 " in v and v.endswith(f"Ap: {psnr:.4f} As: 0.7500")


def test_window_scores_follow_calculate_psnr():
    import numpy as np
    rows = np.zeros((14, 4))
    rows[:, 1] = np.arange(14) * 1000.0
    rows[:, 2] = np.linspace(0.5, 0.9, 14)
    losses = np.arange(15, dtype=np.float32)
    s = T.window_scores(rows, losses, 4, 5)
    assert len(s) == 43 and s[:15] == [float(v) for v in losses]
    assert s[15] == float("inf")                             # utils/util.py: mse == 0 -> inf
    assert s[16] == 20 * math.log10(255.0 / math.sqrt(1000 / 60))
    assert s[29:] == [float(v) for v in rows[:, 2]]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _gloo_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        mine = torch.tensor([float(rank + 1)] * 43 + [2.0 + rank], dtype=torch.float64)
        q.put((rank, T.reduce_sums(mine).tolist()))
    finally:
        dist.destroy_process_group()


def test_val_sums_all_reduce_under_gloo():
    assert T.reduce_sums(torch.ones(3, dtype=torch.float64)).tolist() == [1.0, 1.0, 1.0]   # no process group
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, q)) for r in range(world)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=180) for _ in range(world))
    [p.join(60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    assert res[0][1] == res[1][1] == [3.0] * 43 + [5.0]
