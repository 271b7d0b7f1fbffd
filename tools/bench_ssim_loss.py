"""The 'cb+ssim' criterion (DESIGN §4r) on one GPU, at the train yml's batch (2 x 128x256) and at 8 x 256x256:

  * loss: the 17-term loss forward + backward (14 outputs vs GT and the 3 cycle pairs) with the library's fused
    launches (`pixel_loss(..., "cb+ssim")`), against the same criterion built from torch.nn.functional.conv2d
    (separable 11-tap passes, five moments per term) with autograd, and against the `cb` launches alone;
  * step: the shipped window's training step (zero_grad, window, loss, backward, Adam) with `cb` and with `cb+ssim`,
    alternating in one process, `--rounds` rounds of `--steps` steps each.

Every time is CUDA events on the stream over a window that ends in a synchronise, after warm-up of every shape.
The outputs and targets are seeded device buffers.  The card, its power limit and SM clocks are read in the same
run.  Prints one JSON line per row.

    python tools/bench_ssim_loss.py [--steps 10] [--rounds 3] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import bin_oracle as O  # noqa: E402
from oracle.metrics_oracle import GAUSS11  # noqa: E402

W_SSIM = 0.01


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def timed(fn, steps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / steps


def conv2d_ssim(a, b):
    """Mean SSIM from torch.nn.functional.conv2d: two 1-D passes per moment, autograd for the backward."""
    g = torch.tensor(GAUSS11, dtype=a.dtype, device=a.device)
    n, c, h, w = a.shape

    def filt(x):
        y = torch.nn.functional.conv2d(x.reshape(n * c, 1, h, w), g.view(1, 1, 11, 1))
        return torch.nn.functional.conv2d(y, g.view(1, 1, 1, 11))
    mu1, mu2 = filt(a), filt(b)
    mu1_sq, mu2_sq, mu1_mu2 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1, s2, s12 = filt(a * a) - mu1_sq, filt(b * b) - mu2_sq, filt(a * b) - mu1_mu2
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    return (((2 * mu1_mu2 + c1) * (2 * s12 + c2)) / ((mu1_sq + mu2_sq + c1) * (s1 + s2 + c2))).mean()


def conv2d_loss(outs, gts):
    pairs = list(zip(outs, gts)) + [(outs[i], outs[j]) for i, j in ((1, 7), (5, 9), (2, 8))]
    terms = [torch.sqrt((a - b) ** 2 + 1e-6).mean() + W_SSIM * (1 - conv2d_ssim(a, b)) for a, b in pairs]
    return torch.stack(terms).mean()


def loss_row(B, h, w, steps, rounds):
    from bin_b200.loss import pixel_loss
    g = torch.Generator(device="cuda").manual_seed(1)
    outs = [torch.rand((B, 3, h, w), device="cuda", generator=g).requires_grad_() for _ in range(14)]
    gts = [torch.rand((B, 3, h, w), device="cuda", generator=g) for _ in range(14)]

    def run(kind):
        def f():
            for o in outs:
                o.grad = None
            if kind == "conv2d":
                loss = conv2d_loss(outs, gts)
            else:
                loss, _ = pixel_loss(outs, gts, kind, ssim_weight=W_SSIM)
            loss.backward()
        return f
    fns = {k: run(k) for k in ("cb", "cb+ssim", "conv2d")}
    for f in fns.values():
        f()
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            ms[k].append(timed(f, steps))
    # the fused loss against the conv2d one on these inputs (fp32 both)
    with torch.no_grad():
        got, _ = pixel_loss(outs, gts, "cb+ssim", ssim_weight=W_SSIM)
        ref = conv2d_loss(outs, gts)
    return {"row": "loss_fwd_bwd_17_terms", "batch": f"{B}x3x{h}x{w}",
            **{f"{k}_ms": [round(x, 3) for x in v] for k, v in ms.items()},
            "conv2d_over_fused": round(min(ms["conv2d"]) / min(ms["cb+ssim"]), 2),
            "loss_fused_minus_conv2d": float(got - ref)}


class Step:
    def __init__(self, B, h, w):
        from bin_b200 import rdn
        from bin_b200.optim import Adam
        torch.manual_seed(0)
        net = rdn.bin_stage4_lstm()
        net.load_state_dict(O.synth_state_dict(0))
        self.net = net.cuda().train()
        self.opt = Adam(self.net.parameters(), lr=1e-4, betas=(0.9, 0.99))
        g = torch.Generator(device="cuda").manual_seed(1)
        self.buf = torch.rand((17, B, 3, h, w), device="cuda", generator=g)

    def step(self, kind):
        from bin_b200.loss import pixel_loss
        from bin_b200.train import gt_list
        buf = self.buf
        self.opt.zero_grad(set_to_none=True)
        b = {"LQs": buf[0:6].transpose(0, 1), "GTenh": buf[6:12].transpose(0, 1), "GTinp": buf[12:].transpose(0, 1)}
        outs = self.net(*[b["LQs"][:, k] for k in range(6)])
        loss, _ = pixel_loss(outs, gt_list(b), kind, nframes=6, version=2, ssim_weight=W_SSIM)
        loss.backward()
        self.opt.step()


def step_row(B, h, w, steps, rounds):
    s = Step(B, h, w)
    for k in ("cb", "cb+ssim"):
        s.step(k)
    ms = {"cb": [], "cb+ssim": []}
    for _ in range(rounds):
        for k in ms:
            ms[k].append(timed(lambda: s.step(k), steps))
    res = {"row": "train_step_shipped_window", "batch": f"{B}x3x{h}x{w}",
           **{f"{k}_ms": [round(x, 2) for x in v] for k, v in ms.items()}}
    res["cb_ssim_over_cb"] = round(min(ms["cb+ssim"]) / min(ms["cb"]), 4)
    del s
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ssim_loss: no CUDA device")
    results = []
    for B, h, w in ((2, 128, 256), (8, 256, 256)):
        for fn in (loss_row, step_row):
            res = {**fn(B, h, w, args.steps, args.rounds), "gpu": gpu_info()}
            print(json.dumps(res), flush=True)
            results.append(res)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
