"""Training-batch builder on the GPU (bin_b200.trainset) against the reference's CPU loader.  Prints one JSON line.

* kernel: `bin_train_batch_u8` for a B = 8 batch at 128x256 and 256x256, CUDA events around 200 back-to-back launches
  queued behind a spin kernel (so host enqueue time is not measured); GB/s counts the fp32 bytes written plus the
  uint8 crop bytes read.
* `ds.batch`: wall time of one B = 8 batch including the host draws, ending in a synchronise (median of 50).
* CPU loader: a cv2 restatement of one sample of data/BIN_dataset.py (17 cv2.imread of 352x640 PNGs, float32 / 255,
  crop, fliplr, BGR->RGB, stack) on one core of this host, on uniform-noise frames (slower to decode than video).
* training: B = 8, 256x256 steps (forward, get_loss, backward, Adam) fed by `ds.batches` against steps on one
  fixed resident batch, alternating, CUDA events.
"""
import ctypes as C
import json
import os
import random
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bin_b200 import _lib, rdn  # noqa: E402
from bin_b200.loss import pixel_loss  # noqa: E402
from bin_b200.optim import Adam  # noqa: E402
from bin_b200.trainset import DeviceBINDataset, DeviceClip  # noqa: E402
from oracle import bin_oracle as O  # noqa: E402
from oracle import trainset_oracle as TO  # noqa: E402

GT_ORDER = ["I2", "I4", "I6", "I8", "I3", "I5", "I7", "I4", "I6", "I5", "I10", "I9", "I8", "I7"]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def clips(n=4, T=120):
    """n synthetic 352x640 clips of T sharp frames, blurry frames synthesised on the device."""
    g = torch.Generator(device="cuda").manual_seed(0)
    return [DeviceClip.from_sharp(f"clip{i}", torch.randint(0, 256, (T, 352, 640, 3), generator=g, device="cuda",
                                                            dtype=torch.uint8)) for i in range(n)]


def kernel_time(ds, B, h, w, reps=200):
    drawn = [ds._draw(i % len(ds)) for i in range(B)]
    tab = (_lib.TrainSample * B)()
    for e, (frames, top, left, flip) in zip(tab, [d for d, _ in drawn]):
        for f, t in enumerate(frames):
            e.src[f] = t.data_ptr()
        e.H, e.W, e.top, e.left, e.flip = frames[0].shape[0], frames[0].shape[1], top, left, flip
    out = torch.empty((17, B, 3, h, w), device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    launch = lambda: _lib.check(L.bin_train_batch_u8(tab, B, h, w, out.data_ptr(), B, 0, s))   # noqa: E731
    for _ in range(10):
        launch()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda._sleep(200_000_000)
    e0.record()
    for _ in range(reps):
        launch()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / reps
    nbytes = 17 * B * h * w * (3 * 4 + 3)
    return {"us": round(us, 2), "GB_s": round(nbytes / us / 1e3, 1), "MB_moved": round(nbytes / 1e6, 2)}


def batch_wall(ds, B, reps=50):
    ts = []
    for r in range(reps + 5):
        idx = [(r * B + k) % len(ds) for k in range(B)]
        t0 = time.perf_counter()
        ds.batch(idx)
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return round(statistics.median(ts[5:]) * 1e3, 3)


def cpu_loader_sample(reps=10):
    import cv2
    import numpy as np
    spec = (("GOPR0001", 72, 352, 640, 7, ()),)
    with tempfile.TemporaryDirectory() as root:
        TO.write_tree(root, spec)
        sdir, bdir = os.path.join(root, "train", "GOPR0001"), os.path.join(root, "train_blur", "GOPR0001")
        rng = random.Random(0)
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            order, top, left, flip = TO.draw(rng, 128, 256)
            lq = [cv2.imread(os.path.join(bdir, TO.name(17 + 8 * k) + ".png"), cv2.IMREAD_UNCHANGED) for k in range(6)]
            enh = [cv2.imread(os.path.join(sdir, TO.name(17 + 8 * k) + ".png"), cv2.IMREAD_UNCHANGED) for k in range(6)]
            inp = [cv2.imread(os.path.join(sdir, TO.name(21 + 8 * k) + ".png"), cv2.IMREAD_UNCHANGED) for k in range(5)]
            out = [torch.from_numpy(TO.crop_stack(fr if order else fr[::-1], top, left, flip, 128, 256))
                   for fr in (lq, enh, inp)]
            ts.append(time.perf_counter() - t0)
            assert out[0].shape == (6, 3, 128, 256) and np.isfinite(out[2].numpy()).all()
    return round(statistics.median(ts) * 1e3, 1)


def train_steps(ds, B=8, steps=5, warm=2):
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    net = net.cuda().train()
    opt = Adam(net.parameters(), lr=1e-4, betas=(0.9, 0.99))

    def step(b):
        I = {f"I{2 * k + 1}": b["GTenh"][:, k] for k in range(6)}
        I.update({f"I{2 * k + 2}": b["GTinp"][:, k] for k in range(5)})
        opt.zero_grad(set_to_none=True)
        outs = net(*[b["LQs"][:, k] for k in range(6)])
        loss, _ = pixel_loss(outs, [I[n] for n in GT_ORDER], "l1")
        loss.backward()
        opt.step()

    fixed = ds.batch(list(range(B)))
    fixed = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in fixed.items()}
    sampler = iter(lambda: random.randrange(len(ds)), None)
    it = ds.batches(sampler, B)
    for _ in range(warm):
        step(next(it))
        step(fixed)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    res = {"fed_by_ds_batches": [], "fixed_resident": []}
    for _ in range(2):
        for key in ("fed_by_ds_batches", "fixed_resident"):
            e0.record()
            for _ in range(steps):
                step(next(it) if key == "fed_by_ds_batches" else fixed)
            e1.record()
            torch.cuda.synchronize()
            res[key].append(round(e0.elapsed_time(e1) / steps, 2))
    return res


def main():
    random.seed(0)
    torch.backends.cudnn.benchmark = False
    info = gpu_info()
    cl = clips()
    rec = {"gpu": info, "host_cpus": os.cpu_count(), "host_cpus_usable": len(os.sched_getaffinity(0))}
    for h, w in ((128, 256), (256, 256)):
        ds = DeviceBINDataset(cl, lq_size=(3, h, w))
        rec[f"kernel_B8_{h}x{w}"] = kernel_time(ds, 8, h, w)
        rec[f"ds_batch_B8_{h}x{w}_ms"] = batch_wall(ds, 8)
    rec["cpu_loader_one_sample_128x256_ms_one_core"] = cpu_loader_sample()
    rec["train_step_B8_256x256_ms"] = train_steps(DeviceBINDataset(cl, lq_size=(3, 256, 256)))
    rec["gpu_after"] = gpu_info()
    rec["windows_per_clip"] = len(cl[0].windows())
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
