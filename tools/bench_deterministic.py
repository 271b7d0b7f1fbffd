"""Cost of deterministic training (torch.use_deterministic_algorithms(True), DESIGN.md §4f).

One step is bin_model.optimize_parameters (bin_model.py:130-141): zero_grad, the six-frame window forward, the fused
get_loss (L1, 17 terms), backward and the one-launch Adam step.  Three settings alternate inside one process, so all
see the same card, clock and neighbours:

    off        the default (atomic sums, wgrad grid = SM count)
    det        torch.use_deterministic_algorithms(True): torch also fills every torch.empty with NaN
    det_nofill the same with torch.utils.deterministic.fill_uninitialized_memory = False

Every run prints one JSON line: ms per step (CUDA events over the timed steps, after warm-up) and max_memory_allocated
over the timed steps, next to the card name and power limit.  A separate torch.profiler pass per mode then reports the
summed device time, per step, of the kernels of the three reductions (and of the weight gradients, whose grid the mode
fixes).

    python tools/bench_deterministic.py                  # B = 8 x 256 x 256, 2 warm-ups, 5 timed steps, 2 rounds
    python tools/bench_deterministic.py --B 4 --H 352 --W 640 --modes off,det_nofill
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bin_b200 import rdn  # noqa: E402
from bin_b200.loss import pixel_loss  # noqa: E402
from bin_b200.optim import Adam  # noqa: E402
from oracle import bin_oracle as O  # noqa: E402

GB = 2.0 ** 30
# kernel-name fragments of the reductions the mode changes: (default kernel, deterministic second pass)
KERNELS = {"pixel_loss": ("::pixel_loss_fwd_kernel", "::pixel_loss_reduce_kernel"),
           "bias_grad": ("::p8_bias_grad_kernel", "::bias_grad_reduce_kernel"),
           "convlstm_wgrad": ("::convlstm_bwd_weights_kernel", "::convlstm_wgrad_reduce_kernel"),
           "conv_wgrad": ("::wgrad_kernel", "::wgrad_reduce_kernel")}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30).stdout
        name, power, clock = [s.strip() for s in q.strip().split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unknown ({e})"}


def set_mode(mode):
    torch.use_deterministic_algorithms(mode != "off")
    torch.utils.deterministic.fill_uninitialized_memory = mode != "det_nofill"


class Setup:
    def __init__(self, B, H, W):
        self.B, self.H, self.W = B, H, W
        net = rdn.bin_stage4_lstm()
        net.load_state_dict(O.synth_state_dict(0), strict=True)
        self.net = net.cuda().train()
        self.fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=1234, smooth=True)]
        self.gt = [f.cuda() for f in O.synth_frames(14, B, H, W, seed=4321, smooth=True)]
        self.opt = Adam(self.net.parameters(), lr=1e-4, betas=(0.9, 0.99))      # yml :52-55

    def step(self):
        self.opt.zero_grad(set_to_none=True)
        loss, _ = pixel_loss(self.net(*self.fr), self.gt, "l1")
        loss.backward()
        self.opt.step()
        return loss

    def run(self, mode, steps, warmup):
        set_mode(mode)
        for _ in range(warmup):
            self.step()
        self.opt.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            loss = self.step()
        e1.record()
        torch.cuda.synchronize()
        return {"mode": mode, "B": self.B, "H": self.H, "W": self.W, "steps": steps, "warmup": warmup,
                "ms_per_step": round(e0.elapsed_time(e1) / steps, 2),
                "max_memory_allocated_GB": round(torch.cuda.max_memory_allocated() / GB, 3),
                "loss_last": loss.item(), **card()}

    def kernel_times(self, mode, steps=2):
        """Device time per step of the reduction kernels, from a profiler pass of its own."""
        from torch.profiler import ProfilerActivity, profile
        set_mode(mode)
        self.step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                self.step()
            torch.cuda.synchronize()
        tot = {}
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            for what, (main, second) in KERNELS.items():
                for part, frag in (("main", main), ("reduce", second)):
                    if frag in ev.name:
                        key = f"{what}.{part}"
                        n, us = tot.get(key, (0, 0.0))
                        tot[key] = (n + 1, us + ev.time_range.elapsed_us())
        return {"kernels_of": mode, "B": self.B, "H": self.H, "W": self.W,
                "per_step": {k: {"launches": n // steps, "ms": round(us / steps / 1000.0, 3)} for k, (n, us) in sorted(tot.items())},
                **card()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=8)
    ap.add_argument("--H", type=int, default=256)
    ap.add_argument("--W", type=int, default=256)
    ap.add_argument("--modes", default="off,det,det_nofill")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds over the modes")
    ap.add_argument("--no-kernels", action="store_true", help="skip the profiler pass")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_deterministic: needs a CUDA device")
    modes = a.modes.split(",")
    if any(m not in ("off", "det", "det_nofill") for m in modes):
        sys.exit("bench_deterministic: modes are off, det, det_nofill")
    s = Setup(a.B, a.H, a.W)
    for _ in range(a.rounds):
        for m in modes:
            print(json.dumps(s.run(m, a.steps, a.warmup)), flush=True)
    if not a.no_kernels:
        for m in ("off", "det_nofill"):
            print(json.dumps(s.kernel_times(m)), flush=True)
    set_mode("off")


if __name__ == "__main__":
    main()
