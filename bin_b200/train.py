"""Training BIN from the reference's option file (options/train/train_adobe_stage4.yml), on one GPU or one process per
GPU under torchrun.  The reference never shipped its trainer; this is the loop its INTEGRATION recipe asks a user to
write around bin_model, with every step of the hot path on the GPU:

  * batches: trainset.DeviceBINDataset (BINDataset + create_dataloader, bit for bit), in create_dataloader's order:
    sequential with one process, DistIterSampler under torchrun (restated here as `DistIterSampler`);
  * step: bin_model.optimize_parameters (bin_model.py:130-141): zero_grad, the window on LQs[:, 0..5], loss.pixel_loss
    of the 14 outputs against get_info's GT list with the cycle terms, x pixel_weight, backward, optim.Adam.step;
    pixel_criterion 'cb+ssim' adds train.ssim_weight * (1 - SSIM) to every term (DESIGN §4r);
  * the per-output losses are running sums on the device, read only at print_freq iterations, so an ordinary iteration
    does not synchronise the host with the device;
  * validation every val_freq iterations at batch 1: the 14 losses and their mean, PSNR and SSIM of each output
    (utils/util.py calculate_psnr / calculate_ssim on tensor2img images), windows sharded over the ranks and the sums
    all-reduced; ReduceLROnPlateau steps on the mean validation loss;
  * lr_scheme MultiStepLR or CosineAnnealingLR_Restart (lr_scheduler.py): update_learning_rate(step, warmup_iter)
    before every iteration, step 1-based, so iteration k runs with the scheduler at last_epoch k (DESIGN §4s);
  * checkpoints `<iter>_G.pth` (base_model.save_network) and `<iter>.state` (save_training_state), and resume from
    them at the exact batch, crop and flip the saved run would have drawn next.

Where it departs from the reference: validation crops come from a `random.Random(manual_seed)` made afresh at every
validation, where the reference's validation would draw from the global `random` the training crops draw from.  Every
validation then scores the same crops, and validating does not change the training batches.

With --cuda_graph (one GPU only) iteration 1 runs eagerly, on a side stream, and the step is then captured once in a
CUDA graph -- zero_grad, the window, the loss, backward, Adam(capturable=True) and the running loss sums -- and
replayed for every later iteration, the batch built into the graph's static input in place (DESIGN §4p).  The bits
are the eager run's.  BIN_B200_GRAPH=0 turns capture off.

python -m bin_b200.train -opt <yml> [--checkpointing recompute] [--max_grad_norm X] [--skip_nonfinite]
[--deterministic] [--from_sharp] [--arch G0,D] [--cuda_graph]; under torchrun each rank trains on its own GPU."""
from __future__ import annotations

import argparse
import logging
import math
import os
import random
import re
import sys
import warnings
from dataclasses import dataclass, field
from typing import Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import rdn
from ._lib import BIN_TRAIN_FRAMES, BinB200Error
from .evaluate import load_weights
from .loss import CB_SSIM, cycle_pairs_for, pixel_loss, pixel_ssim_loss
from .lr_scheduler import CosineAnnealingLR_Restart, MultiStepLR_Restart, warm_up
from .metrics import image_metrics_batch
from .optim import Adam
from .streaming import tensor2img_u8
from .trainset import DeviceBINDataset, DeviceClip

NOUT = 14
PLATEAU, MULTISTEP, COSINE = "ReduceLROnPlateau", "MultiStepLR", "CosineAnnealingLR_Restart"
# bin_model.get_info (nframes 6, bin_model.py:530-534): output k is scored against I_GT_OF[k]; feed_data maps I(2m+1) to
# GTenh[:, m] and I(2m) to GTinp[:, m-1] (bin_model.py:164-174)
I_GT_OF = (2, 4, 6, 8, 3, 5, 7, 4, 6, 5, 10, 9, 8, 7)
IGNORED = ("gpu_ids", "datasets.train.n_workers", "datasets.val.n_workers")
LOG_FORMAT = logging.Formatter('%(asctime)s.%(msecs)03d - %(levelname)s: %(message)s', datefmt='%y-%m-%d %H:%M:%S')


# ----------------------------------------------------------------------------- options
@dataclass
class Options:
    """The keys of a train yml this driver honours (options/train/train_adobe_stage4.yml)."""
    name: str
    train_root: str                      # datasets.train.dataroot_LQ
    train_mode: str                      # datasets.train.name: <root>/<mode>, <mode>_blur, <mode>_list
    batch_size: int                      # global: batch_size // world per rank
    train_lq_size: Tuple[int, int, int]
    use_shuffle: bool                    # read; create_dataloader passes shuffle=False whatever it says
    val_root: Optional[str]              # None: no datasets.val, no validation
    val_mode: Optional[str]
    val_lq_size: Optional[Tuple[int, int, int]]
    version: int
    pretrain_model_G: Optional[str]
    strict_load: bool
    resume_state: Optional[str]
    save_path: str
    lr: float
    beta1: float
    beta2: float
    weight_decay: float
    pixel_criterion: str
    pixel_weight: float
    factor: Optional[float]              # ReduceLROnPlateau only (None with the other schemes)
    patience: Optional[int]
    epochs: int
    val_freq: int
    manual_seed: int
    print_freq: int
    save_freq: int
    ignored: List[str] = field(default_factory=list)
    ssim_weight: Optional[float] = None   # train.ssim_weight: read, and required, with pixel_criterion cb+ssim only
    lr_scheme: str = PLATEAU               # train.lr_scheme (DESIGN §4s); the keys below are read with MultiStepLR and
    lr_steps: Optional[List[int]] = None   # CosineAnnealingLR_Restart only
    lr_gamma: Optional[float] = None
    clear_state: bool = False
    T_period: Optional[List[int]] = None
    eta_min: Optional[float] = None
    restarts: Optional[List[int]] = None   # as the yml gives them (None: unset); a restart r happens at iteration r + 1
    restart_weights: Optional[List[float]] = None
    warmup_iter: int = -1

    @property
    def experiments_root(self) -> str:
        return os.path.join(self.save_path, "experiments", self.name)      # options.parse

    @property
    def models_dir(self) -> str:
        return os.path.join(self.experiments_root, "models")

    @property
    def state_dir(self) -> str:
        return os.path.join(self.experiments_root, "training_state")


def _get(opt: dict, key: str, default=KeyError):
    node = opt
    for part in key.split("."):
        if not isinstance(node, dict) or part not in node:
            if default is KeyError:
                raise BinB200Error(f"train options: {key} is missing")
            return default
        node = node[part]
    return node


def _path(p) -> Optional[str]:
    return None if p in (None, "") else os.path.expanduser(str(p))


def _schedule_options(opt: dict, scheme: str) -> dict:
    """The keys of MultiStepLR / CosineAnnealingLR_Restart, checked so that no configuration on which
    bin_model's scheduler would fail part-way through training starts (DESIGN §4s)."""
    def need(key: str):
        v = _get(opt, "train." + key, None)
        if v is None:
            raise BinB200Error(f"train.{key} is missing: train.lr_scheme {scheme} needs it")
        return v

    def ints(key: str, v) -> List[int]:
        if not isinstance(v, (list, tuple)):
            raise BinB200Error(f"train.{key} must be a list (train.lr_scheme {scheme}), got {v!r}")
        return [int(float(x)) for x in v]

    restarts, weights = _get(opt, "train.restarts", None), _get(opt, "train.restart_weights", None)
    restarts = ints("restarts", restarts) if restarts is not None else None
    if weights is not None and not isinstance(weights, (list, tuple)):
        raise BinB200Error(f"train.restart_weights must be a list (train.lr_scheme {scheme}), got {weights!r}")
    weights = [float(w) for w in weights] if weights is not None else None
    n_restarts, n_weights = len(restarts or [0]), len(weights or [1])       # unset or empty: one restart, weight 1
    if n_restarts != n_weights:
        raise BinB200Error(f"train.restarts ({n_restarts} restart(s)) and train.restart_weights ({n_weights} "
                           f"weight(s)) differ in length: train.lr_scheme {scheme} pairs them")
    out = dict(lr_scheme=scheme, restarts=restarts, restart_weights=weights,
               warmup_iter=int(float(_get(opt, "train.warmup_iter", -1))))
    if scheme == MULTISTEP:
        out.update(lr_steps=ints("lr_steps", need("lr_steps")), lr_gamma=float(need("lr_gamma")),
                   clear_state=bool(_get(opt, "train.clear_state", False)))
    else:
        T_period = ints("T_period", need("T_period"))
        if len(T_period) < n_restarts + 1:
            raise BinB200Error(f"train.T_period has {len(T_period)} entr{'y' if len(T_period) == 1 else 'ies'}; "
                               f"train.lr_scheme {scheme} with {n_restarts} restart(s) needs {n_restarts + 1}"
                               + ("" if restarts else " (with train.restarts unset, iteration 1 is a restart)"))
        out.update(T_period=T_period, eta_min=float(need("eta_min")))
    return out


def parse_options(opt: dict) -> Options:
    """The honoured keys of a parsed train yml.  Raises BinB200Error naming the key for what this driver does not do:
    another model than bin_stage4, nframes other than 6, an lr_scheme other than ReduceLROnPlateau, MultiStepLR and
    CosineAnnealingLR_Restart or one missing a key it needs, ft_tsa_only, an unknown pixel_criterion, cb+ssim without
    train.ssim_weight."""
    if _get(opt, "network_G.which_model_G") != "bin_stage4":
        raise BinB200Error(f"network_G.which_model_G: {_get(opt, 'network_G.which_model_G')!r} is not trained here; "
                           "only bin_stage4 is")
    if int(_get(opt, "network_G.nframes")) != 6:
        raise BinB200Error("network_G.nframes: only 6 (the 14-output bin_stage4 window) is trained here")
    scheme = _get(opt, "train.lr_scheme")
    if scheme not in (PLATEAU, MULTISTEP, COSINE):
        raise BinB200Error(f"train.lr_scheme: {scheme!r} is not supported; {PLATEAU}, {MULTISTEP} and {COSINE} are "
                           "(bin_model.py:103-125)")
    schedule = _schedule_options(opt, scheme) if scheme != PLATEAU else {}
    if _get(opt, "train.ft_tsa_only", None):
        raise BinB200Error("train.ft_tsa_only is not supported")
    crit = _get(opt, "train.pixel_criterion")
    if crit not in ("l1", "l2", "cb", CB_SSIM):
        raise BinB200Error(f"train.pixel_criterion: {crit!r} is not one of l1, l2, cb (bin_model.py:54-61) or "
                           f"{CB_SSIM}")
    ssim_weight = float(_get(opt, "train.ssim_weight")) if crit == CB_SSIM else None
    val = _get(opt, "datasets.val", None)
    return Options(
        name=str(_get(opt, "name")),
        train_root=_path(_get(opt, "datasets.train.dataroot_LQ")),
        train_mode=str(_get(opt, "datasets.train.name")),
        batch_size=int(_get(opt, "datasets.train.batch_size")),
        train_lq_size=tuple(int(v) for v in _get(opt, "datasets.train.LQ_size")),
        use_shuffle=bool(_get(opt, "datasets.train.use_shuffle", False)),
        val_root=_path(_get(opt, "datasets.val.dataroot_LQ")) if val else None,
        val_mode=str(_get(opt, "datasets.val.name")) if val else None,
        val_lq_size=tuple(int(v) for v in _get(opt, "datasets.val.LQ_size")) if val else None,
        version=int(_get(opt, "network_G.version")),
        pretrain_model_G=_path(_get(opt, "path.pretrain_model_G", None)),
        strict_load=bool(_get(opt, "path.strict_load", True)),
        resume_state=_path(_get(opt, "path.resume_state", None)),
        save_path=_path(_get(opt, "path.save_path")),
        lr=float(_get(opt, "train.lr_G")),
        beta1=float(_get(opt, "train.beta1")),
        beta2=float(_get(opt, "train.beta2")),
        weight_decay=float(_get(opt, "train.weight_decay_G", 0) or 0),     # bin_model.py:65
        pixel_criterion=crit,
        pixel_weight=float(_get(opt, "train.pixel_weight")),
        factor=float(_get(opt, "train.factor")) if scheme == PLATEAU else None,
        patience=int(_get(opt, "train.patience")) if scheme == PLATEAU else None,
        epochs=int(_get(opt, "train.epoch")),
        val_freq=int(float(_get(opt, "train.val_freq"))),
        manual_seed=int(_get(opt, "train.manual_seed")),
        print_freq=int(float(_get(opt, "logger.print_freq"))),
        save_freq=int(float(_get(opt, "logger.save_checkpoint_freq"))),
        ignored=[k for k in IGNORED if _get(opt, k, None) is not None],
        ssim_weight=ssim_weight,
        **schedule)


def load_options(path: str) -> Options:
    import yaml
    with open(path) as fh:
        return parse_options(yaml.safe_load(fh))


# ----------------------------------------------------------------------------- order and schedule
class DistIterSampler:
    """data/data_sampler.py DistIterSampler over a dataset of n samples: each epoch, randperm(total_size) seeded by the
    epoch, every index % n, then rank, rank + world, ... (total_size = world * ceil(n * ratio / world))."""

    def __init__(self, n: int, world: int, rank: int, ratio: int = 100):
        self.n, self.world, self.rank, self.epoch = n, world, rank, 0
        self.num_samples = int(math.ceil(n * ratio / world))
        self.total_size = self.num_samples * world

    def set_epoch(self, epoch: int) -> None:
        self.epoch = epoch

    def __iter__(self) -> Iterator[int]:
        g = torch.Generator()
        g.manual_seed(self.epoch)
        idx = [v % self.n for v in torch.randperm(self.total_size, generator=g).tolist()]
        return iter(idx[self.rank:self.total_size:self.world])

    def __len__(self) -> int:
        return self.num_samples


class SequentialSampler:
    """create_dataloader with one process: shuffle=False, so each epoch walks the (once shuffled) dataset in order."""

    def __init__(self, n: int):
        self.n = n

    def set_epoch(self, epoch: int) -> None:
        pass

    def __iter__(self) -> Iterator[int]:
        return iter(range(self.n))

    def __len__(self) -> int:
        return self.n


def make_sampler(n: int, world: int, rank: int, ratio: int = 100):
    return SequentialSampler(n) if world == 1 else DistIterSampler(n, world, rank, ratio)


def per_rank_batch(batch_size: int, world: int) -> int:
    if batch_size % world:
        raise BinB200Error(f"datasets.train.batch_size {batch_size} is not divisible by the {world} ranks "
                           "(create_dataloader asserts it)")
    return batch_size // world


def events(step: int, print_freq: int, val_freq: int, save_freq: int) -> Tuple[str, ...]:
    """What runs after iteration `step` (1-based): 'print', 'val', 'save', in that order."""
    return tuple(k for k, f in (("print", print_freq), ("val", val_freq), ("save", save_freq)) if f > 0 and step % f == 0)


def resume_position(state_epoch: int, state_iter: int, iters_per_epoch: int) -> Tuple[int, int]:
    """-> (epoch, batches of it already run) after `state_iter` iterations of `iters_per_epoch` each, from epoch 0.
    A state saved after the last batch of epoch e says epoch e and resumes at batch 0 of epoch e + 1."""
    if iters_per_epoch < 1:
        raise BinB200Error("resume: an epoch of this dataset has no full batch")
    epoch, done = divmod(state_iter, iters_per_epoch)
    if state_epoch != (epoch - 1 if done == 0 and state_iter > 0 else epoch):
        raise BinB200Error(f"resume: iteration {state_iter} is in epoch {epoch} at {iters_per_epoch} iterations per "
                           f"epoch, but the state says epoch {state_epoch}; the dataset or batch size differs from "
                           "the saved run's")
    return epoch, done


def gt_list(batch: Dict) -> List[torch.Tensor]:
    """get_info(mode=1)'s GT list of a DeviceBINDataset batch."""
    return [batch["GTenh"][:, i // 2] if i % 2 else batch["GTinp"][:, i // 2 - 1] for i in I_GT_OF]


# ----------------------------------------------------------------------------- logs
def train_message(epoch: int, step: int, lr: float, avg: Sequence[float], guard: Optional[Tuple[int, float]],
                  ssim_loss: Optional[float] = None) -> str:
    """avg: the 14 per-output losses and their mean (get_current_log('train')'s '0'..'13', 'Al'), averaged since the
    last message; guard: (skipped steps, last grad norm) when the step is guarded; ssim_loss: with cb+ssim, the SSIM
    part of the loss (ssim_weight * (1 - SSIM), the mean over the 14 outputs; Video_base_model's 'ssim_loss')."""
    msg = "<epoch:{:3d}, iter:{:8,d}, lr:{:.3e}> ".format(epoch, step, lr)
    msg += "".join("{:s}: {:.4e} ".format(k, v) for k, v in zip([str(i) for i in range(NOUT)] + ["Al"], avg))
    if ssim_loss is not None:
        msg += "ssim_loss: {:.4e} ".format(ssim_loss)
    if guard is not None:
        skipped, norm = guard
        msg += "skipped: {:d} grad_norm: {} ".format(skipped, "n/a" if norm is None else "{:.4e}".format(norm))
    return msg.rstrip()


def val_log(sums: Sequence[float]):
    """get_current_log('val') from the reduced sums [14 losses, mean loss, 14 PSNR, 14 SSIM, window count]:
    -> (avg_log_dict, avg_psnr_dict, mean PSNR, mean SSIM, mean loss)."""
    sums = [float(v) for v in sums]
    n = sums[-1]
    loss, psnr, ssim = sums[:NOUT + 1], sums[NOUT + 1:2 * NOUT + 1], sums[2 * NOUT + 1:3 * NOUT + 1]
    avg_log = {"Al" + str(i): loss[i] / n for i in range(NOUT)}
    avg_log["Al"] = loss[NOUT] / n
    avg_psnr = {"Ap" + str(i): psnr[i] / n for i in range(NOUT)}
    psnr_mean = sum(psnr[i] / n for i in range(NOUT)) / NOUT
    avg_psnr["Ap"] = psnr_mean
    return avg_log, avg_psnr, psnr_mean, sum(ssim[i] / n for i in range(NOUT)) / NOUT, loss[NOUT] / n


def val_message(epoch: int, step: int, log) -> str:
    avg_log, avg_psnr, _, ssim_mean, _ = log
    msg = "<epoch:{:3d}, iter:{:8,d}> # Validation # ".format(epoch, step)
    msg += "".join("{:s}: {:.4e} ".format(k, v) for k, v in avg_log.items())
    msg += "".join("{:s}: {:.4f} ".format(k, v) for k, v in avg_psnr.items())
    return msg + "As: {:.4f}".format(ssim_mean)


def window_scores(rows: np.ndarray, losses: np.ndarray, h: int, w: int) -> List[float]:
    """One validation window's terms, as the reference's meters take them: rows (14, 4) float64 of image_metrics_batch
    (sum |a-b|, sum (a-b)^2, Gaussian SSIM, box SSIM) of each output against its GT; losses (15,) float32 (14 + mean).
    -> [14 losses, mean loss, 14 calculate_psnr, 14 calculate_ssim] as Python floats."""
    n = h * w * 3
    psnr = []
    for r in rows:
        mse = int(r[1]) / n                                 # utils/util.py:201-208, as metrics.calculate_psnr
        psnr.append(float('inf') if mse == 0 else 20 * math.log10(255.0 / math.sqrt(mse)))
    return [float(v) for v in losses] + psnr + [float(np.float64(r[2])) for r in rows]


def reduce_sums(sums: torch.Tensor) -> torch.Tensor:
    """All-reduce (sum) a float64 tensor over the ranks of the initialised process group, in place."""
    if torch.distributed.is_available() and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1:
        torch.distributed.all_reduce(sums)
    return sums


# ----------------------------------------------------------------------------- data
def _from_sharp_tree(root: str, mode: str, device, lq_size, rng) -> DeviceBINDataset:
    """Clips built by DeviceClip.from_sharp from <root>/<mode>/<folder> alone, folders in os.listdir order."""
    import cv2
    clips = []
    for folder in os.listdir(os.path.join(root, mode)):
        d = os.path.join(root, mode, folder)
        names = sorted(os.listdir(d))
        want = [str(k).zfill(5) + ".png" for k in range(1, len(names) + 1)]
        if names != want:
            raise BinB200Error(f"--from_sharp: the sharp frames of {d} must be named 00001.png, 00002.png, ...")
        imgs = []
        for nm in names:
            img = cv2.imread(os.path.join(d, nm), cv2.IMREAD_UNCHANGED)
            if img is None or img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] < 3:
                raise BinB200Error(f"--from_sharp: {os.path.join(d, nm)} is not an 8-bit colour image")
            imgs.append(torch.from_numpy(np.ascontiguousarray(img[:, :, :3])))
        clips.append(DeviceClip.from_sharp(folder, torch.stack(imgs).to(device)))
    return DeviceBINDataset(clips, lq_size=lq_size, rng=rng)


def build_dataset(root: str, mode: str, device, lq_size, rng, from_sharp: bool) -> DeviceBINDataset:
    if from_sharp:
        return _from_sharp_tree(root, mode, device, lq_size, rng)
    return DeviceBINDataset.from_tree(root, mode=mode, device=device, lq_size=lq_size, rng=rng)


def make_scheduler(opt: torch.optim.Optimizer, o: Options):
    """bin_model.__init__'s scheduler for the yml's lr_scheme (bin_model.py:103-125)."""
    if o.lr_scheme == MULTISTEP:
        return MultiStepLR_Restart(opt, o.lr_steps, restarts=o.restarts, weights=o.restart_weights, gamma=o.lr_gamma,
                                   clear_state=o.clear_state)
    if o.lr_scheme == COSINE:
        return CosineAnnealingLR_Restart(opt, o.T_period, restarts=o.restarts, weights=o.restart_weights,
                                         eta_min=o.eta_min)
    return torch.optim.lr_scheduler.ReduceLROnPlateau(opt, "min", factor=o.factor, patience=o.patience)


def scheduler_kind(sd: dict) -> str:
    """The lr_scheme whose scheduler wrote the state dict `sd` (its class's own keys tell them apart)."""
    if "T_period" in sd:
        return COSINE
    if "milestones" in sd and "restart_weights" in sd:
        return MULTISTEP
    if "patience" in sd and "factor" in sd:
        return PLATEAU
    return "unknown"


def graph_mode(requested: bool, world: int) -> bool:
    """Whether a run captures its training step: asked for, and not turned off by BIN_B200_GRAPH=0 (as inference's
    window graph is).  Refused with more than one rank: the step of a DistributedDataParallel run all-reduces through
    NCCL, which this driver does not capture."""
    if requested and world > 1:
        raise BinB200Error(f"--cuda_graph trains on one GPU; this run has {world} ranks (DistributedDataParallel's NCCL "
                           "all-reduce is not captured)")
    return requested and rdn._graphs_enabled()


# ----------------------------------------------------------------------------- the driver
class Trainer:
    """One rank's training run.  `run()` trains to the end of the yml's epochs (or `max_iters` iterations in all);
    `net` is the unwrapped module, `opt` the optimizer, `scheduler` the yml's lr_scheme (make_scheduler).

    rank / world default to the initialised process group, else (0, 1); the device is cuda:<LOCAL_RANK> under a
    process group, else the current device.  sync_debug: a torch.cuda.set_sync_debug_mode level under which every
    iteration after the first (batch, step, running sums) runs, for checking that it never waits on the device.
    cuda_graph: capture the step after the first iteration and replay it (see the module docstring, `graph_mode`)."""

    def __init__(self, opts: Options, *, checkpointing: Optional[str] = None, max_grad_norm: Optional[float] = None,
                 skip_nonfinite: bool = False, deterministic: bool = False, from_sharp: bool = False,
                 arch: Optional[Tuple[int, int]] = None, ratio: int = 100, sync_debug: Optional[str] = None,
                 stdout: bool = True, cuda_graph: bool = False):
        self.o = opts
        dist = torch.distributed.is_available() and torch.distributed.is_initialized()
        self.rank = torch.distributed.get_rank() if dist else 0
        self.world = torch.distributed.get_world_size() if dist else 1
        self.dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")) if dist else torch.cuda.current_device())
        self.sync_debug = sync_debug
        self.cuda_graph = graph_mode(cuda_graph, self.world)
        self.log = logging.Logger(f"bin_b200.train.{id(self)}", logging.INFO)
        if self.rank == 0:
            os.makedirs(opts.models_dir, exist_ok=True)
            os.makedirs(opts.state_dir, exist_ok=True)
            for h in [logging.FileHandler(os.path.join(opts.experiments_root, f"train_{opts.name}.log"), mode="a")] + \
                     ([logging.StreamHandler(sys.stdout)] if stdout else []):
                h.setFormatter(LOG_FORMAT)
                self.log.addHandler(h)
        for k in opts.ignored:
            self.log.info(f"{k} is ignored: one process per GPU under torchrun, batches are built on the GPU")
        if deterministic:
            torch.use_deterministic_algorithms(True)
            torch.utils.deterministic.fill_uninitialized_memory = False     # every workspace byte read is written
        self.B = per_rank_batch(opts.batch_size, self.world)

        random.seed(opts.manual_seed)
        torch.manual_seed(opts.manual_seed)
        with torch.cuda.device(self.dev):
            self.train_set = build_dataset(opts.train_root, opts.train_mode, self.dev, opts.train_lq_size, random,
                                           from_sharp)
            self.val_set = None
            if opts.val_root is not None:
                self.val_set = build_dataset(opts.val_root, opts.val_mode, self.dev, opts.val_lq_size,
                                             random.Random(opts.manual_seed), from_sharp)
        self.sampler = make_sampler(len(self.train_set), self.world, self.rank, ratio)
        self.iters_per_epoch = len(self.sampler) // self.B
        if self.iters_per_epoch < 1:
            raise BinB200Error(f"{len(self.train_set)} training windows make no batch of {self.B} per rank")
        self.log.info(f"Training {opts.name}: {len(self.train_set)} windows, batch {opts.batch_size} over {self.world} "
                      f"rank(s), {self.iters_per_epoch} iterations per epoch, {opts.epochs} epochs")

        net = rdn.bin_stage4_lstm()
        if arch is not None:
            net.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=arch[0], D=arch[1])
        if opts.pretrain_model_G and not opts.resume_state:
            load_weights(net, opts.pretrain_model_G, strict=opts.strict_load)
            self.log.info(f"Loading model for G [{opts.pretrain_model_G:s}] ...")
        self.net = net.to(self.dev).train()
        if checkpointing is not None:
            rdn.set_activation_checkpointing(self.net, checkpointing)
        params = []
        for k, v in self.net.named_parameters():
            if v.requires_grad:
                params.append(v)
            else:
                self.log.warning(f"Params [{k:s}] will not optimize.")
        self.opt = Adam(params, lr=opts.lr, weight_decay=opts.weight_decay, betas=(opts.beta1, opts.beta2),
                        max_grad_norm=max_grad_norm, skip_nonfinite=skip_nonfinite, capturable=self.cuda_graph)
        if cuda_graph and not self.cuda_graph:
            self.log.info("BIN_B200_GRAPH=0: the training step runs eagerly")
        self.guarded = max_grad_norm is not None or skip_nonfinite
        self.scheduler = make_scheduler(self.opt, opts)
        self.model = self.net
        if self.world > 1:
            from torch.nn.parallel import DistributedDataParallel
            self.model = DistributedDataParallel(self.net, device_ids=[self.dev.index])   # bin_model.py:39-41

        self.step = 0
        if opts.resume_state:
            self._resume(opts.resume_state)
        self.ssim = opts.pixel_criterion == CB_SSIM
        self._ssim_part: Optional[torch.Tensor] = None
        with torch.cuda.device(self.dev):     # 14 losses, their mean and, with cb+ssim, the SSIM part
            self.loss_sums = torch.zeros(NOUT + 1 + self.ssim, dtype=torch.float32, device=self.dev)
        self.loss_count = 0
        # --cuda_graph: the static batch buffer every batch is built into, then the graph and what it owns
        self._static: Optional[torch.Tensor] = None
        self._graph: Optional[torch.cuda.CUDAGraph] = None
        self._graph_keep: tuple = ()

    # ------------------------------------------------------------------ checkpoints
    def _resume(self, path: str) -> None:
        state = torch.load(path, map_location=self.dev)
        weights = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(path))), "models",
                               "{}_G.pth".format(state["iter"]))
        load_weights(self.net, weights, strict=True)
        if len(state["optimizers"]) != 1 or len(state["schedulers"]) != 1:
            raise BinB200Error(f"resume: {path} holds {len(state['optimizers'])} optimizers and "
                               f"{len(state['schedulers'])} schedulers; this driver has one of each")
        saved = scheduler_kind(state["schedulers"][0])
        if saved != self.o.lr_scheme:
            raise BinB200Error(f"resume: {path} holds a {saved} scheduler, but the yml's train.lr_scheme is "
                               f"{self.o.lr_scheme}")
        self.opt.load_state_dict(state["optimizers"][0])
        self.scheduler.load_state_dict(state["schedulers"][0])
        resume_position(int(state["epoch"]), int(state["iter"]), self.iters_per_epoch)
        self.step = int(state["iter"])
        # the crops and flips of the samples the saved run drew (every iteration draws for B samples)
        self.train_set.skip_draws(self.step * self.B)
        self.log.info(f"Resuming training from epoch: {self.epoch}, iter: {self.step} ({weights}).")

    def save(self) -> None:
        """base_model.save_network and save_training_state at the current iteration (rank 0 writes)."""
        opt_sd, sch_sd = self.opt.state_dict(), self.scheduler.state_dict()
        if self.rank != 0:
            return
        sd = self.net.state_dict()
        for k, v in sd.items():
            sd[k] = v.cpu()
        torch.save(sd, os.path.join(self.o.models_dir, "{}_G.pth".format(self.step)))
        torch.save({"epoch": self.epoch, "iter": self.step, "schedulers": [sch_sd], "optimizers": [opt_sd]},
                   os.path.join(self.o.state_dir, "{}.state".format(self.step)))
        self.log.info("Saving models and training states.")

    # ------------------------------------------------------------------ one iteration
    def _loss(self, outs, batch: Dict) -> Tuple[torch.Tensor, List[torch.Tensor]]:
        """The criterion of the yml on the 14 outputs.  With cb+ssim it also leaves the step's SSIM part (the mean
        over the 14 outputs of ssim_weight * (1 - SSIM)) in self._ssim_part, on the device."""
        if not self.ssim:
            return pixel_loss(outs, gt_list(batch), self.o.pixel_criterion, nframes=6, version=self.o.version)
        loss, losses, means = pixel_ssim_loss(outs, gt_list(batch), self.o.ssim_weight,
                                              cycle_pairs=cycle_pairs_for(6, self.o.version))
        self._ssim_part = self.o.ssim_weight * (1.0 - torch.stack(means).mean())
        return loss, losses

    def _sums_row(self, loss: torch.Tensor, losses: List[torch.Tensor]) -> torch.Tensor:
        return torch.stack(list(losses) + [loss.detach()] + ([self._ssim_part] if self.ssim else []))

    def train_step(self, batch: Dict) -> Tuple[torch.Tensor, List[torch.Tensor]]:
        """bin_model.optimize_parameters on one batch: -> (loss, the 14 per-output losses), on the device."""
        self.opt.zero_grad(set_to_none=True)
        outs = self.model(*[batch["LQs"][:, k] for k in range(6)])
        loss, losses = self._loss(outs, batch)
        (self.o.pixel_weight * loss).backward()
        self.opt.step()
        return loss, losses

    def _iterate(self, batch: Dict) -> None:
        """One training iteration on `batch`, the running loss sums included: eager, or a replay of the captured step
        (the first iteration of a --cuda_graph run is its eager warm-up, and the capture follows it)."""
        if not self.cuda_graph:
            loss, losses = self.train_step(batch)
            self.loss_sums += self._sums_row(loss, losses)
        elif self._graph is not None:
            self.opt.replay(self._graph)
        else:
            self._warm_up_and_capture(batch)

    def _warm_up_and_capture(self, batch: Dict) -> None:
        """Run `batch` eagerly on a side stream (a real step, with the eager bits; it also makes the tables, the packed
        weights and the kernels' shared-memory opt-ins), then capture one step on the static batch buffer.  A capture
        records without running, so it applies no update.  The gradients stay the warm-up's tensors: zero_grad(
        set_to_none=False) inside the graph, and backward accumulates into them.  The graph owns the scratch workspaces
        the side stream and the capture allocated."""
        side = torch.cuda.Stream(self.dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            loss, losses = self.train_step(batch)
            self.loss_sums += self._sums_row(loss, losses)
            rdn.take_workspace(self.dev)
        torch.cuda.current_stream().wait_stream(side)
        graph, capture = torch.cuda.CUDAGraph(), torch.cuda.Stream(self.dev)
        with torch.cuda.graph(graph, stream=capture):
            self.opt.zero_grad(set_to_none=False)
            outs = self.model(*[batch["LQs"][:, k] for k in range(6)])
            loss, losses = self._loss(outs, batch)
            (self.o.pixel_weight * loss).backward()
            self.opt.step()
            self.loss_sums += self._sums_row(loss, losses)
            ws = rdn.take_workspace(self.dev)
        del outs, loss, losses
        self._ssim_part = None
        self._graph, self._graph_keep = graph, (ws, capture)

    def _batches(self) -> Iterator[Dict]:
        """The batches of the epoch the next iteration is in, from the next one on (with --cuda_graph, each built into
        the one static batch buffer the captured step reads)."""
        epoch, done = divmod(self.step, self.iters_per_epoch)
        self.sampler.set_epoch(epoch)
        it = iter(self.sampler)
        for _ in range(done * self.B):
            next(it)
        if self.cuda_graph and self._static is None:
            h, w = self.train_set.h, self.train_set.w
            self._static = torch.empty((BIN_TRAIN_FRAMES, self.B, 3, h, w), dtype=torch.float32, device=self.dev)
        return self.train_set.batches(it, self.B, self._static)

    def run(self, max_iters: Optional[int] = None) -> None:
        """Train to the end of the last epoch, or until `max_iters` iterations in all have run."""
        o = self.o
        end = o.epochs * self.iters_per_epoch
        if max_iters is not None:
            end = min(end, max_iters)
        saved, first = None, True
        with torch.cuda.device(self.dev):
            while self.step < end:
                batches = self._batches()
                for _ in range(min(end, (self.step // self.iters_per_epoch + 1) * self.iters_per_epoch) - self.step):
                    mode = torch.cuda.get_sync_debug_mode()
                    if self.sync_debug is not None and not first:
                        torch.cuda.set_sync_debug_mode(self.sync_debug)
                    try:
                        if o.lr_scheme != PLATEAU:
                            self._update_learning_rate()
                        self._iterate(next(batches))
                    finally:
                        torch.cuda.set_sync_debug_mode(mode)
                    first = False
                    self.step += 1
                    self.loss_count += 1
                    ev = events(self.step, o.print_freq, o.val_freq, o.save_freq)
                    if "print" in ev:
                        self._print()
                    if "val" in ev and self.val_set is not None:
                        log = self.validate()
                        if o.lr_scheme == PLATEAU:
                            self.scheduler.step(log[4])
                        self.log.info(val_message(self.epoch, self.step, log))
                    if "save" in ev:
                        self.save()
                        saved = self.step
            if saved != self.step:
                self.save()
            torch.cuda.synchronize(self.dev)
        self.log.info("End of training.")

    def _update_learning_rate(self) -> None:
        """base_model.update_learning_rate(step, warmup_iter) before iteration `step` (1-based) runs: the scheduler
        steps to last_epoch == step, then the warm-up.  The loop steps the scheduler before the optimizer on purpose,
        so torch's warning about that order is not shown."""
        with warnings.catch_warnings():
            warnings.filterwarnings("ignore", message=re.escape("Detected call of `lr_scheduler.step()` before"))
            self.scheduler.step()
        warm_up(self.opt, self.step + 1, self.o.warmup_iter)

    @property
    def epoch(self) -> int:
        """The epoch of the last iteration run (0 before the first)."""
        return max(self.step - 1, 0) // self.iters_per_epoch

    def _print(self) -> None:
        avg = [v / self.loss_count for v in self.loss_sums.tolist()]
        guard = None
        if self.guarded:
            self.opt.resolve()
            guard = (self.opt.skipped_steps, self.opt.last_grad_norm)
        self.log.info(train_message(self.epoch, self.step, self.opt.param_groups[0]["lr"], avg[:NOUT + 1], guard,
                                    avg[NOUT + 1] if self.ssim else None))
        self.loss_sums.zero_()
        self.loss_count = 0

    # ------------------------------------------------------------------ validation
    @torch.no_grad()
    def validate(self) -> tuple:
        """The val split at batch 1, this rank's share of its windows (i = rank, rank + world, ...), the crops drawn
        from a fresh random.Random(manual_seed) for every window in order.  -> get_current_log('val') of the sums over
        all ranks (val_log)."""
        vs = self.val_set
        vs.rng = random.Random(self.o.manual_seed)
        rows, losses = [], []
        for i in range(len(vs)):
            if i % self.world != self.rank:
                vs.skip_draws(1)
                continue
            b = vs.batch([i])
            outs = self.net(*[b["LQs"][:, k] for k in range(6)])
            loss, lst = self._loss(outs, b)
            pairs = [(tensor2img_u8(outs[k][0]), tensor2img_u8(g[0])) for k, g in enumerate(gt_list(b))]
            rows.append(image_metrics_batch(pairs))
            losses.append(torch.stack(lst + [loss]))
        sums = [0] * (3 * NOUT + 1)                          # AverageMeter: sum += val, in window order
        if rows:
            h, w = vs.h, vs.w
            for r, l in zip(torch.stack(rows).cpu().numpy(), torch.stack(losses).cpu().numpy()):
                for k, v in enumerate(window_scores(r, l, h, w)):
                    sums[k] += v
        t = torch.tensor(sums + [len(rows)], dtype=torch.float64, device=self.dev)
        self.val_sums = reduce_sums(t).tolist()
        return val_log(self.val_sums)

    def close(self) -> None:
        for h in list(self.log.handlers):
            h.close()
            self.log.removeHandler(h)


# ----------------------------------------------------------------------------- command line
def _arch(v: str) -> Tuple[int, int]:
    try:
        g0, d = (int(x) for x in v.split(","))
    except ValueError:
        raise argparse.ArgumentTypeError(f"--arch takes G0,D (e.g. 64,6), got {v!r}") from None
    return g0, d


def main(argv=None) -> None:
    ap = argparse.ArgumentParser(description="Train bin_stage4 from a train yml of the reference (one process per GPU "
                                             "under torchrun)")
    ap.add_argument("-opt", required=True, help="e.g. options/train/train_adobe_stage4.yml")
    ap.add_argument("--checkpointing", choices=("recompute",), default=None,
                    help="rebuild each backbone stage's activations in its backward")
    ap.add_argument("--max_grad_norm", type=float, default=None, help="clip the gradients by their global norm")
    ap.add_argument("--skip_nonfinite", action="store_true", help="skip a step with an inf or NaN gradient")
    ap.add_argument("--deterministic", action="store_true", help="torch.use_deterministic_algorithms(True)")
    ap.add_argument("--from_sharp", action="store_true",
                    help="synthesise the blurry frames from <root>/<mode>/<folder> (DeviceClip.from_sharp)")
    ap.add_argument("--arch", type=_arch, default=None, help="backbone G0,D of a light window, e.g. 64,6")
    ap.add_argument("--ratio", type=int, default=100, help="DistIterSampler's epoch enlargement under torchrun")
    ap.add_argument("--cuda_graph", action="store_true",
                    help="capture the training step in a CUDA graph after the first iteration and replay it (one GPU)")
    args = ap.parse_args(argv)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    graph_mode(args.cuda_graph, world)
    opts = load_options(args.opt)

    distributed = world > 1
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if distributed:
        torch.distributed.init_process_group("nccl", device_id=torch.device("cuda", local))
    try:
        t = Trainer(opts, checkpointing=args.checkpointing, max_grad_norm=args.max_grad_norm,
                    skip_nonfinite=args.skip_nonfinite, deterministic=args.deterministic, from_sharp=args.from_sharp,
                    arch=args.arch, ratio=args.ratio, cuda_graph=args.cuda_graph)
        try:
            t.run()
        finally:
            t.close()
    finally:
        if distributed:
            torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
