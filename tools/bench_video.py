"""Time one video the way test.py walks it: per-window module calls on test_py_window's frame lists against
stream_video.  Prints the card, its power limit and SM clocks, read in the same run.

    python tools/bench_video.py [--frames 20] [--size 768x1344] [--rounds 3] [--out path.json]

A video of --frames synthetic frames (B = 1, fp16 mode, synthetic weights), already on the device as fp32 frames padded
the way test.py pads 720p (768x1344).  Both paths give test.py's N-1 windows with all 14 outputs, and drop them:
  per-window  net(*[F[j] for j in test_py_window(i, N)]) for i = 0 .. N-2, on the module's CUDA-graph path: 17 backbone
              calls per window, 17 (N-1) in all.
  stream      stream_video(net, F): each stage-1 frame pair once per video, 13 N - 11 calls in all.
The paths alternate, one whole video each, for --rounds rounds after one warm-up video each.  windows/s is N-1 over the
video's time between CUDA events; the table gives the median and the range.  Memory: torch.cuda.memory_allocated()
before the path's last video (frames, weights, cached workspace and graph), and max_memory_allocated() growth above it
during that video.
Needs a CUDA device; there is no CPU fallback."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bin_b200 import _lib, rdn                                   # noqa: E402
from bin_b200.streaming import stream_video, test_py_window      # noqa: E402
from oracle import bin_oracle as O                               # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        name, power, sm, sm_max = [s.strip() for s in r.stdout.strip().split(",")]
    except Exception as e:  # noqa: BLE001
        name, power, sm, sm_max = torch.cuda.get_device_name(), f"unknown ({e})", "unknown", "unknown"
    return {"name": name, "power_limit": power, "sm_clock": sm, "max_sm_clock": sm_max}


def per_window(net, video):
    n = len(video)
    for i in range(n - 1):
        net(*[video[j] for j in test_py_window(i, n)])
    return (n - 1) * sum(1 for node in rdn._window_live(range(14)) if node[0] != "lstm")     # 17 per window


def streamed(net, video):
    stream = stream_video(net, video)
    for _ in stream:
        pass
    return stream.backbone_calls


def timed(fn, net, video):
    """(ms for the video, backbone calls, resident bytes before, peak growth in bytes)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    calls = fn(net, video)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), calls, base, torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--size", default="768x1344")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_video: needs a CUDA device (the window has no CPU path)")
    _lib.check(_lib.lib().bin_check_device())
    H, W = (int(v) for v in args.size.split("x"))
    n = args.frames
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    net = net.cuda().eval()
    video = [f.cuda() for f in O.synth_frames(n, 1, H, W, seed=11, smooth=True)]
    out = {"card_before": card(), "frames": n, "windows": n - 1, "H": H, "W": W, "B": 1, "precision": "fp16"}
    paths = {"per_window": per_window, "stream": streamed}
    runs = {k: [] for k in paths}
    with torch.no_grad():
        for r in range(args.rounds + 1):                # round 0 warms up: weight packs, workspace, graph capture
            for name, fn in paths.items():
                res = timed(fn, net, video)
                if r:
                    runs[name].append(res)
    for name, rs in runs.items():
        rates = [(n - 1) / (ms / 1e3) for ms, _, _, _ in rs]
        _, calls, base, peak = rs[-1]
        out[name] = {"windows_per_s": statistics.median(rates), "range": [min(rates), max(rates)],
                     "backbone_calls": calls, "resident_bytes": base, "peak_growth_bytes": peak}
    out["card_after"] = card()
    pw, st = out["per_window"], out["stream"]
    print(f"{n}-frame video, {n - 1} windows, {H}x{W}, B=1, fp16, {args.rounds} rounds")
    for name, r in (("per-window", pw), ("stream", st)):
        print(f"  {name:10s} {r['windows_per_s']:.2f} windows/s [{r['range'][0]:.2f}, {r['range'][1]:.2f}], "
              f"{r['backbone_calls']} backbone calls, resident {r['resident_bytes'] / 1e9:.3f} GB, "
              f"peak growth {r['peak_growth_bytes'] / 1e9:.3f} GB")
    print(f"  stream / per-window: {st['windows_per_s'] / pw['windows_per_s']:.3f} "
          f"(calls {pw['backbone_calls']} / {st['backbone_calls']} = {pw['backbone_calls'] / st['backbone_calls']:.3f})")
    c = out["card_after"]
    print(f"card: {c['name']}, power limit {c['power_limit']}, SM clock {out['card_before']['sm_clock']} -> {c['sm_clock']}"
          f" (max {c['max_sm_clock']})")
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
