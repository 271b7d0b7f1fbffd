"""Step time and peak memory of a training step in the two activation modes (rdn.set_activation_checkpointing).

One step is bin_model.optimize_parameters (bin_model.py:130-141): zero_grad, the six-frame window forward, the fused
get_loss (L1, 17 terms), backward and the one-launch Adam step.  Modes alternate inside one process, so both see the
same card, clock and neighbours.  Every run prints one JSON line: ms per step (CUDA events over the timed steps, after
warm-up) and max_memory_allocated over the timed steps, next to the card name and power limit.

    python tools/bench_train_memory.py 8 256 256                 # both modes, alternating
    python tools/bench_train_memory.py 8 352 640 --modes recompute
    python tools/bench_train_memory.py 8 256 256 --plan 352 640  # also predict the peaks at 352x640 (see plan())
    python tools/bench_train_memory.py 8 256 256 --breakdown     # where the default step's peak goes (separate run)

--plan H W takes, from the runs at the first size, the memory that the size queries do not account for, assumes it
grows with B*H*W, and prints the predicted peak of both modes at H x W and the largest B of each mode that fits in
80 % of the memory free at start.  Run the chosen batches as separate invocations: nothing is sized by trial
allocation, and a fresh process does not inherit the other runs' cached blocks.  --breakdown records the allocator's history (torch.cuda.memory._record_memory_history) during one default
step, replays it to the moment of the peak, and groups the live bytes by the line of bin_b200 that allocated them.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bin_b200 import _lib, rdn  # noqa: E402
from bin_b200.loss import pixel_loss  # noqa: E402
from bin_b200.optim import Adam  # noqa: E402
from oracle import bin_oracle as O  # noqa: E402

STAGES = ((2, 5), (3, 6), (5, 4), (5, 2))       # (frames per call, calls) of the window's four batched stages
GB = 2.0 ** 30


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30).stdout
        name, power, clock = [s.strip() for s in q.strip().split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unknown ({e})"}


def sizes(B, H, W):
    """Bytes from the library's size queries: saved activations of the default mode (S), the largest inference
    workspace of one stage (what the recompute mode holds) and the largest gradient workspace of one stage."""
    L = _lib.lib()
    S = sum(L.bin_backbone_train_workspace_bytes(n, B * c, H, W) for n, c in STAGES)
    inf = max(L.bin_backbone_workspace_bytes(n, B * c, H, W) for n, c in STAGES)
    gws = max(L.bin_backbone_grad_workspace_bytes(n, B * c, H, W) for n, c in STAGES)
    return S, inf, gws


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
        rdn.release_workspaces()
        torch.cuda.empty_cache()                  # the other mode's cached blocks would fragment this mode's large ones
        rdn.set_activation_checkpointing(self.net, mode)
        for _ in range(warmup):
            self.step()
        self.opt.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        resident = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            loss = self.step()
        e1.record()
        torch.cuda.synchronize()
        S, inf, gws = sizes(self.B, self.H, self.W)
        return {"mode": mode or "default", "B": self.B, "H": self.H, "W": self.W, "steps": steps, "warmup": warmup,
                "ms_per_step": round(e0.elapsed_time(e1) / steps, 2),
                "max_memory_allocated_GB": round(torch.cuda.max_memory_allocated() / GB, 3),
                "held_before_step_GB": round(resident / GB, 3), "saved_activations_S_GB": round(S / GB, 3),
                "stage_inference_ws_GB": round(inf / GB, 3), "stage_grad_ws_GB": round(gws / GB, 3),
                "loss_last": loss.item(), **card()}

    def close(self):
        del self.net, self.fr, self.gt, self.opt
        rdn.release_workspaces()
        torch.cuda.empty_cache()


def breakdown(setup):
    """Replay one default step's allocator history to its peak; group the live bytes by allocating line."""
    rdn.release_workspaces()
    rdn.set_activation_checkpointing(setup.net, None)
    setup.step()
    setup.opt.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    torch.cuda.memory._record_memory_history(max_entries=2_000_000, stacks="python")
    setup.step()
    torch.cuda.synchronize()
    snap = torch.cuda.memory._snapshot()
    torch.cuda.memory._record_memory_history(enabled=None)
    peak_stat = torch.cuda.max_memory_allocated()

    def site(frames):
        for f in frames:
            fn = f.get("filename", "")
            if ("bin_b200" in fn or "bench_train_memory" in fn) and "site-packages" not in fn:
                return f"{os.path.relpath(fn, ROOT)}:{f['line']} {f['name']}"
        return "other (" + (frames[0]["name"] if frames else "?") + ")"

    trace = snap["device_traces"][torch.cuda.current_device()]
    live, cur, peak, at_peak = {}, base, base, {}
    for e in trace:
        if e["action"] == "alloc":
            live[e["addr"]] = (e["size"], site(e.get("frames", [])))
            cur += e["size"]
            if cur > peak:
                peak, at_peak = cur, dict(live)
        elif e["action"] == "free_completed" and e["addr"] in live:
            cur -= live.pop(e["addr"])[0]
    groups = {}
    for size, where in at_peak.values():
        n, tot = groups.get(where, (0, 0))
        groups[where] = (n + 1, tot + size)
    S, inf, gws = sizes(setup.B, setup.H, setup.W)
    out = {"breakdown": "default mode, one step", "B": setup.B, "H": setup.H, "W": setup.W,
           "held_before_step_GB": round(base / GB, 3), "peak_replayed_GB": round(peak / GB, 3),
           "max_memory_allocated_GB": round(peak_stat / GB, 3), "saved_activations_S_GB": round(S / GB, 3),
           "stage_grad_ws_GB": round(gws / GB, 3),
           "live_at_peak": [{"site": k, "tensors": n, "GB": round(t / GB, 3)}
                            for k, (n, t) in sorted(groups.items(), key=lambda kv: -kv[1][1])], **card()}
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("B", type=int)
    ap.add_argument("H", type=int)
    ap.add_argument("W", type=int)
    ap.add_argument("--modes", default="default,recompute")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=2, help="alternating rounds over the modes")
    ap.add_argument("--plan", type=int, nargs=2, metavar=("H", "W"))
    ap.add_argument("--breakdown", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_train_memory: needs a CUDA device")
    modes = [None if m == "default" else m for m in a.modes.split(",")]
    free0, total = torch.cuda.mem_get_info()
    s = Setup(a.B, a.H, a.W)
    if a.breakdown:
        breakdown(s)
        s.close()
        return
    rows = []
    for _ in range(a.repeats):
        for m in modes:
            r = s.run(m, a.steps, a.warmup)
            rows.append(r)
            print(json.dumps(r), flush=True)
    s.close()
    if a.plan:
        plan(rows, a, free0, total)


def plan(rows, a, free0, total):
    """Predict both modes' peaks at the --plan size from the size queries and the overhead measured here.

    Default: every stage's training workspace (S) is alive when the backward starts, and the first backward (stage 4,
    two 5-frame calls) adds its gradient workspace.  Recompute: one stage's inference workspace is held throughout
    (it is part of the memory held before the step), and the largest stage gradient workspace adds to it.  The rest --
    outputs, loss and frame gradients, ConvLSTM buffers -- is measured at this size per item-pixel and scaled."""
    batch_bytes = lambda B, H, W: 20 * B * 3 * H * W * 4          # the 6 frames + 14 targets, resident across steps
    px = a.B * a.H * a.W
    S, inf, gws = sizes(a.B, a.H, a.W)
    gws4 = _lib.lib().bin_backbone_grad_workspace_bytes(5, 2 * a.B, a.H, a.W)
    d = next(r for r in rows if r["mode"] == "default")
    r = next(r for r in rows if r["mode"] == "recompute")
    held_fixed = d["held_before_step_GB"] * GB - batch_bytes(a.B, a.H, a.W)   # weights and Adam state
    ov_d = (d["max_memory_allocated_GB"] * GB - d["held_before_step_GB"] * GB - S - gws4) / px
    ov_r = (r["max_memory_allocated_GB"] * GB - r["held_before_step_GB"] * GB - gws) / px
    H2, W2 = a.plan
    budget = 0.8 * free0

    def predict(mode, B):
        S2, inf2, gws2 = sizes(B, H2, W2)
        base = held_fixed + batch_bytes(B, H2, W2)
        if mode is None:
            return base + S2 + _lib.lib().bin_backbone_grad_workspace_bytes(5, 2 * B, H2, W2) + ov_d * B * H2 * W2
        return base + inf2 + gws2 + ov_r * B * H2 * W2

    b_both = max((B for B in range(1, 129) if predict(None, B) <= budget), default=0)
    b_rc = max((B for B in range(1, 129) if predict("recompute", B) <= budget), default=0)
    print(json.dumps({"plan": f"{H2}x{W2}", "free_at_start_GB": round(free0 / GB, 2), "total_GB": round(total / GB, 2),
                      "budget_GB": round(budget / GB, 2), "overhead_bytes_per_item_pixel": [round(ov_d, 1), round(ov_r, 1)],
                      "B_both_modes": b_both, "B_recompute_only": b_rc,
                      "predicted_GB": {f"{m or 'default'}@B={B}": round(predict(m, B) / GB, 2)
                                       for m in (None, "recompute") for B in sorted({8, b_both, b_rc})}}), flush=True)


if __name__ == "__main__":
    main()
