"""Iterations per second of the training driver (bin_b200.train.Trainer) against the bare step loop it wraps
(DeviceBINDataset.batches -> module -> pixel_loss -> backward -> optim.Adam.step, as tests/test_gpu_train_driver.py
writes it), at the train yml's shapes (batch 2, 128x256) and at batch 8 x 256x256, on the same GPU in one process.

The data is a seeded PNG tree written to a temporary directory (4 training folders x 12 blurry frames = 28 windows, one
validation folder of 7 windows), the weights synthetic.  Driver and bare loop alternate, after one warm-up run of each;
each timed run is --steps iterations and ends in a device synchronise.  Checkpoint writes are left out of the driver's
timed runs (they happen every save_checkpoint_freq iterations, 5000 in the yml).  Also reported: the host CPU seconds
per iteration (process time over the run) and one validation's wall time, as a share of the wall time of val_freq
iterations plus that validation.  Prints one JSON line (and writes it to --json when given).

    python tools/bench_train_driver.py [--steps 30] [--repeats 3] [--val_freq 10000] [--json out.json]
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import bin_oracle as O  # noqa: E402

H, W, FIRST = 352, 640, 17


def make_tree(root, mode, folders, nb, seed):
    import cv2
    g = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, mode + "_list"), exist_ok=True)
    for f in folders:
        for sub in (mode, mode + "_blur"):
            os.makedirs(os.path.join(root, sub, f))
        base = g.integers(0, 256, size=(H // 8, W // 8, 3)).astype(np.float32)
        names = []
        for m in range(2 * nb - 1):
            base += g.normal(0, 3, size=base.shape).astype(np.float32)
            img = np.clip(cv2.resize(base, (W, H), interpolation=cv2.INTER_CUBIC), 0, 255).astype(np.uint8)
            cv2.imwrite(os.path.join(root, mode, f, f"{FIRST + 4 * m:05d}.png"), img)
            if m % 2 == 0:
                names.append(f"{FIRST + 4 * m:05d}.png")
                cv2.imwrite(os.path.join(root, mode + "_blur", f, names[-1]), cv2.GaussianBlur(img, (9, 9), 3.0))
        with open(os.path.join(root, mode + "_list", f + "_im_list.txt"), "w") as fh:
            fh.write("\n".join(names))


def options(root, save, weights, batch, lq):
    return {
        "name": "bench", "gpu_ids": [0],
        "datasets": {"train": {"name": "train", "dataroot_LQ": root, "use_shuffle": True, "batch_size": batch,
                               "LQ_size": [3, lq[0], lq[1]]},
                     "val": {"name": "test", "dataroot_LQ": root, "LQ_size": [3, lq[0], lq[1]]}},
        "network_G": {"which_model_G": "bin_stage4", "nframes": 6, "version": 2},
        "path": {"pretrain_model_G": weights, "save_path": save, "strict_load": True, "resume_state": None},
        "train": {"lr_G": 1e-4, "lr_scheme": "ReduceLROnPlateau", "beta1": 0.9, "beta2": 0.99, "factor": 0.2,
                  "patience": 1, "epoch": 1000000, "pixel_criterion": "cb", "pixel_weight": 1.0, "val_freq": 1e9,
                  "manual_seed": 0},
        "logger": {"print_freq": 100, "save_checkpoint_freq": 1e9},
    }


class Bare:
    """The step loop without the driver: batches in dataset order, epoch after epoch."""

    def __init__(self, root, weights, batch, lq):
        from bin_b200 import rdn
        from bin_b200.evaluate import load_weights
        from bin_b200.optim import Adam
        from bin_b200.trainset import DeviceBINDataset
        random.seed(0)
        torch.manual_seed(0)
        self.ds = DeviceBINDataset.from_tree(root, mode="train", device="cuda", lq_size=(3,) + lq)
        net = rdn.bin_stage4_lstm()
        load_weights(net, weights)
        self.net = net.cuda().train()
        self.opt = Adam(self.net.parameters(), lr=1e-4, betas=(0.9, 0.99))
        self.batch = batch
        self.it = iter(())

    def _next(self):
        b = next(self.it, None)
        if b is None:
            self.it = self.ds.batches(range(len(self.ds)), self.batch)
            b = next(self.it)
        return b

    def run(self, steps):
        from bin_b200.loss import pixel_loss
        from bin_b200.train import gt_list
        for _ in range(steps):
            b = self._next()
            self.opt.zero_grad(set_to_none=True)
            outs = self.net(*[b["LQs"][:, k] for k in range(6)])
            loss, _ = pixel_loss(outs, gt_list(b), "cb", nframes=6, version=2)
            (1.0 * loss).backward()
            self.opt.step()
        torch.cuda.synchronize()


def timed(fn):
    torch.cuda.synchronize()
    w0, c0 = time.perf_counter(), time.process_time()
    fn()
    return time.perf_counter() - w0, time.process_time() - c0


def bench_shape(root, save, weights, batch, lq, steps, repeats, val_freq):
    from bin_b200 import train as T
    t = T.Trainer(T.parse_options(options(root, save, weights, batch, lq)), stdout=False)
    t.save = lambda: None
    bare = Bare(root, weights, batch, lq)
    t.run(max_iters=t.step + steps)                         # warm-up: packs, workspaces, Adam tables
    bare.run(steps)
    drv, brw, dcpu, bcpu = [], [], [], []
    for _ in range(repeats):
        w, c = timed(lambda: t.run(max_iters=t.step + steps))
        drv.append(w / steps)
        dcpu.append(c / steps)
        w, c = timed(lambda: bare.run(steps))
        brw.append(w / steps)
        bcpu.append(c / steps)
    t.validate()                                            # warm-up: the inference graph at this shape
    vals = [timed(t.validate)[0] for _ in range(2)]
    t.close()
    it_d, it_b, val = statistics.median(drv), statistics.median(brw), min(vals)
    return {"batch": batch, "crop": list(lq), "driver_it_s": round(1 / it_d, 3), "bare_it_s": round(1 / it_b, 3),
            "driver_overhead_pct": round(100 * (it_d / it_b - 1), 2),
            "driver_ms_runs": [round(1e3 * x, 2) for x in drv], "bare_ms_runs": [round(1e3 * x, 2) for x in brw],
            "driver_cpu_s_per_it": round(statistics.median(dcpu), 4), "bare_cpu_s_per_it": round(statistics.median(bcpu), 4),
            "val_windows": len(t.val_set), "val_s": round(val, 3),
            "val_share_pct_at_val_freq": round(100 * val / (val + val_freq * it_d), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--val_freq", type=int, default=10000)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_driver: no CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "tree")
        make_tree(root, "train", [f"clip{k}" for k in range(4)], 12, 1)
        make_tree(root, "test", ["val0"], 12, 2)
        weights = os.path.join(tmp, "w.pth")
        torch.save(O.synth_state_dict(0), weights)
        rows = [bench_shape(root, os.path.join(tmp, f"s{b}"), weights, b, lq, args.steps, args.repeats, args.val_freq)
                for b, lq in ((2, (128, 256)), (8, (256, 256)))]
    out = {"gpu": gpu[0] if gpu else torch.cuda.get_device_name(), "cpus": os.cpu_count(), "steps": args.steps,
           "val_freq": args.val_freq, "rows": rows}
    line = json.dumps(out)
    print(line)
    if args.json:
        with open(args.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
