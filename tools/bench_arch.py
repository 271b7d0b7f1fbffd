"""Speed of the shipped window (G0 = 96, D = 12) against the reference's default configuration (G0 = 64, D = 6, the light
window: net.model = RDN_residual_interp_5_input(lstm=True, GO=64, D=6)), in one process, alternating the two.

  inference  windows/s of the six-frame window at 1280x720 (batch 1, fp16, graphed, all 14 outputs)
  training   ms per step at batch 8 x 256x256: forward, fused L1 get_loss, backward and the Adam step

Prints the card's name and power limit with the numbers, and the MAC ratio of the two backbones (from their shapes), as
one JSON line.  Usage: python tools/bench_arch.py [--rounds R] [--windows N] [--steps S]"""
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
from oracle import arch_oracle as A  # noqa: E402
from oracle import bin_oracle as O  # noqa: E402

ARCHS = {"96x12": (96, 12), "64x6": (64, 6)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30).stdout
        name, power = [s.strip() for s in q.strip().split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unknown ({e})"}


def backbone_macs_per_position(nframes, g0, d):
    """MACs per low-resolution position of one backbone call, from its conv shapes (UPNet.2 runs at 4 positions)."""
    macs = 0
    for name, shape in A.backbone_param_shapes(nframes, g0, d):
        if name.endswith("weight"):
            co, ci, k, _ = shape
            macs += co * ci * k * k * (4 if name.startswith("UPNet.2") else 1)
    return macs


def build(g0, d, train):
    net = rdn.bin_stage4_lstm()
    if (g0, d) != (96, 12):
        net.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=g0, D=d)
    net.load_state_dict(A.synth_state_dict(0, g0, d), strict=True)
    net = net.cuda()
    return net.train() if train else net.eval()


def time_windows(net, frames, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        e0.record()
        for _ in range(n):
            net(*frames)
        e1.record()
    torch.cuda.synchronize()
    return n / (e0.elapsed_time(e1) / 1e3)


def time_steps(net, opt, fr, gt, n):
    def step():
        opt.zero_grad(set_to_none=True)
        loss, _ = pixel_loss(net(*fr), gt, "l1")
        loss.backward()
        opt.step()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--windows", type=int, default=20)
    ap.add_argument("--steps", type=int, default=5)
    a = ap.parse_args()
    res = {"card": card(), "windows_per_s_1280x720": {k: [] for k in ARCHS}, "train_ms_b8_256": {k: [] for k in ARCHS}}
    res["backbone_macs_per_position"] = {k: {n: backbone_macs_per_position(n, *v) for n in (2, 3, 5)} for k, v in ARCHS.items()}

    frames = [f.cuda() for f in O.synth_frames(6, 1, 720, 1280, seed=1234, smooth=True)]
    nets = {k: build(*v, train=False) for k, v in ARCHS.items()}
    for net in nets.values():                          # warm-up: weight packs, graph capture
        time_windows(net, frames, 3)
    for _ in range(a.rounds):
        for k, net in nets.items():
            res["windows_per_s_1280x720"][k].append(round(time_windows(net, frames, a.windows), 3))
    del nets, frames
    torch.cuda.empty_cache()

    fr = [f.cuda() for f in O.synth_frames(6, 8, 256, 256, seed=1234, smooth=True)]
    gt = [f.cuda() for f in O.synth_frames(14, 8, 256, 256, seed=4321, smooth=True)]
    nets = {k: build(*v, train=True) for k, v in ARCHS.items()}
    opts = {k: Adam(net.parameters(), lr=1e-4, betas=(0.9, 0.99)) for k, net in nets.items()}
    for k in ARCHS:
        time_steps(nets[k], opts[k], fr, gt, 2)
    for _ in range(a.rounds):
        for k in ARCHS:
            res["train_ms_b8_256"][k].append(round(time_steps(nets[k], opts[k], fr, gt, a.steps), 2))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
