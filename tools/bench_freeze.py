"""Training steps with part of the network frozen (requires_grad False, DESIGN.md §4g).

One step is bin_model.optimize_parameters (bin_model.py:130-141) as a fine-tuning run drives it: zero_grad, the
six-frame window forward, the fused get_loss (L1, 17 terms), backward, and the one-launch Adam step over the trainable
tensors only (bin_model builds its optimizer from the requires_grad parameters, bin_model.py:89-95).  The configurations
alternate inside one process, so all see the same card, clock and neighbours:

    all            every tensor trainable
    stage1_frozen  model1_1 (stage 1, 5 of the 17 backbone calls) frozen
    only_model4_1  only model4_1 (stage 4, 2 calls) trainable
    only_convlstm  only the six ConvLSTM cells trainable

Every run prints one JSON line: ms per step (CUDA events over the timed steps, after warm-up) and max_memory_allocated
over the timed steps, next to the card name, power limit and maximum SM clock.  A profiler pass per configuration then
reports the launches per step of the weight-gradient, bias-gradient, ConvLSTM weight-pass and fused-RDB-tail kernels.

    python tools/bench_freeze.py                         # B = 8 x 256 x 256, 2 warm-ups, 5 timed steps, 2 rounds
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
CONFIGS = {"all": lambda k: True,
           "stage1_frozen": lambda k: not k.startswith("model.model1_1."),
           "only_model4_1": lambda k: k.startswith("model.model4_1."),
           "only_convlstm": lambda k: ".Gates." in k}
KERNELS = {"wgrad": "::wgrad_kernel", "bias_grad": "::p8_bias_grad_kernel",
           "convlstm_wgrad": "::convlstm_bwd_weights_kernel", "rdb_tail": "::rdb_tail_kernel"}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30).stdout
        name, power, clock = [s.strip() for s in q.strip().split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unknown ({e})"}


class Setup:
    def __init__(self, B, H, W):
        self.B, self.H, self.W = B, H, W
        net = rdn.bin_stage4_lstm()
        net.load_state_dict(O.synth_state_dict(0), strict=True)
        self.net = net.cuda().train()
        self.fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=1234, smooth=True)]
        self.gt = [f.cuda() for f in O.synth_frames(14, B, H, W, seed=4321, smooth=True)]
        self.opts = {}

    def use(self, config):
        for k, p in self.net.named_parameters():
            p.requires_grad_(CONFIGS[config](k))
        if config not in self.opts:                              # yml :52-55, trainable tensors only
            self.opts[config] = Adam([p for p in self.net.parameters() if p.requires_grad], lr=1e-4, betas=(0.9, 0.99))
        return self.opts[config]

    def step(self, opt):
        opt.zero_grad(set_to_none=True)
        self.net.zero_grad(set_to_none=True)
        loss, _ = pixel_loss(self.net(*self.fr), self.gt, "l1")
        loss.backward()
        opt.step()
        return loss

    def run(self, config, steps, warmup):
        rdn.release_workspaces()                 # the shared inference workspace counts only where a config uses it
        opt = self.use(config)
        for _ in range(warmup):
            self.step(opt)
        self.net.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            loss = self.step(opt)
        e1.record()
        torch.cuda.synchronize()
        return {"config": config, "B": self.B, "H": self.H, "W": self.W, "steps": steps, "warmup": warmup,
                "ms_per_step": round(e0.elapsed_time(e1) / steps, 2),
                "max_memory_allocated_GB": round(torch.cuda.max_memory_allocated() / GB, 3),
                "loss_last": loss.item(), **card()}

    def launches(self, config):
        from torch.profiler import ProfilerActivity, profile
        opt = self.use(config)
        self.step(opt)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            self.step(opt)
            torch.cuda.synchronize()
        n = dict.fromkeys(KERNELS, 0)
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                for key, frag in KERNELS.items():
                    n[key] += frag in ev.name
        return {"launches_of": config, "B": self.B, "H": self.H, "W": self.W, "per_step": n}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=8)
    ap.add_argument("--H", type=int, default=256)
    ap.add_argument("--W", type=int, default=256)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds over the configurations")
    ap.add_argument("--no-launches", action="store_true", help="skip the profiler pass")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_freeze: needs a CUDA device")
    configs = a.configs.split(",")
    if any(c not in CONFIGS for c in configs):
        sys.exit(f"bench_freeze: configurations are {', '.join(CONFIGS)}")
    s = Setup(a.B, a.H, a.W)
    for _ in range(a.rounds):
        for c in configs:
            print(json.dumps(s.run(c, a.steps, a.warmup)), flush=True)
    if not a.no_launches:
        for c in configs:
            print(json.dumps(s.launches(c)), flush=True)


if __name__ == "__main__":
    main()
