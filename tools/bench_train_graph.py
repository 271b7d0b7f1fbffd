"""Training step eager against the same step captured in a CUDA graph (DESIGN §4p), in one process on one GPU: the
train yml's batch (2 x 128x256, pixel_criterion cb) and 8 x 256x256, on the shipped window and the light G0 = 64, D = 6
one.

One net per row.  The graph is captured after an eager warm-up step, as the driver does; eager iterations run the plain
optimizer's step with fresh gradients (the graph's static gradients are set aside meanwhile, so its tables stay
valid).  The two alternate, `--rounds` rounds of `--steps` iterations each, every round timed with CUDA events on the
stream.  The batch is a seeded device buffer: the batch build is the same host work in both modes and is left out.
A separate profiled pass of 3 iterations per mode sums the kernel time per iteration; the GPU-busy fraction is that
over the timed ms per iteration.  The card, its power limit and SM clocks are read in the same run.  Prints one JSON
line per row.

    python tools/bench_train_graph.py [--steps 20] [--rounds 2] [--rows all|yml] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import arch_oracle as A  # noqa: E402
from oracle import bin_oracle as O  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


class Row:
    def __init__(self, arch, B, h, w):
        from bin_b200 import rdn
        from bin_b200.optim import Adam
        torch.manual_seed(0)
        net = rdn.bin_stage4_lstm()
        if arch == "light":
            net.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=64, D=6)
            net.load_state_dict(A.synth_state_dict(0, 64, 6))
        else:
            net.load_state_dict(O.synth_state_dict(0))
        self.net = net.cuda().train()
        self.params = list(self.net.parameters())
        self.eager_opt = Adam(self.params, lr=1e-4, betas=(0.9, 0.99))
        self.graph_opt = Adam(self.params, lr=1e-4, betas=(0.9, 0.99), capturable=True)
        g = torch.Generator(device="cuda").manual_seed(1)
        self.static = torch.rand((17, B, 3, h, w), device="cuda", generator=g)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self._step(self.graph_opt, True)
            rdn.take_workspace(self.static.device)
        torch.cuda.current_stream().wait_stream(side)
        self.graph, self.capture = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        with torch.cuda.graph(self.graph, stream=self.capture):
            self._step(self.graph_opt, False)
            self.ws = rdn.take_workspace(self.static.device)
        self.eager()                                        # warm-up of the eager path (its own optimizer tables)

    def _step(self, opt, set_to_none):
        from bin_b200.loss import pixel_loss
        from bin_b200.train import gt_list
        buf = self.static
        opt.zero_grad(set_to_none=set_to_none)
        b = {"LQs": buf[0:6].transpose(0, 1), "GTenh": buf[6:12].transpose(0, 1), "GTinp": buf[12:].transpose(0, 1)}
        outs = self.net(*[b["LQs"][:, k] for k in range(6)])
        loss, _ = pixel_loss(outs, gt_list(b), "cb", nframes=6, version=2)
        loss.backward()
        opt.step()

    def eager(self):
        kept = [p.grad for p in self.params]
        for p in self.params:
            p.grad = None
        self._step(self.eager_opt, True)
        for p, g in zip(self.params, kept):
            p.grad = g

    def graphed(self):
        self.graph_opt.replay(self.graph)


def timed(fn, steps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / steps


def kernel_ms(fn, steps=3):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    total = sum(ev.self_device_time_total for ev in prof.key_averages())
    return total / 1000.0 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--rows", choices=("all", "yml"), default="all")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_graph: no CUDA device")
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    rows = [("shipped", 2, 128, 256), ("light", 2, 128, 256)]
    if args.rows == "all":
        rows += [("shipped", 8, 256, 256), ("light", 8, 256, 256)]
    results = []
    for arch, B, h, w in rows:
        r = Row(arch, B, h, w)
        ms = {"eager": [], "graph": []}
        for _ in range(args.rounds):
            ms["eager"].append(timed(r.eager, args.steps))
            ms["graph"].append(timed(r.graphed, args.steps))
        busy = {k: kernel_ms(f) for k, f in (("eager", r.eager), ("graph", r.graphed))}
        res = {"window": arch, "batch": f"{B}x{h}x{w}", "gpu": gpu_info(),
               "eager_ms": [round(x, 2) for x in ms["eager"]], "graph_ms": [round(x, 2) for x in ms["graph"]],
               "eager_kernel_ms": round(busy["eager"], 2), "graph_kernel_ms": round(busy["graph"], 2)}
        res["eager_busy"] = round(busy["eager"] / min(ms["eager"]), 3)
        res["graph_busy"] = round(busy["graph"] / min(ms["graph"]), 3)
        res["speedup"] = round(min(ms["eager"]) / min(ms["graph"]), 3)
        print(json.dumps(res), flush=True)
        results.append(res)
        del r
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
