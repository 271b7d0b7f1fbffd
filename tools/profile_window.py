"""Per-layer attribution of the six-frame window: where the device time of bench.py's workload goes, layer by layer,
against each layer's floor.

    python tools/profile_window.py [--height 720] [--width 1280] [--windows 5] [--warmup 3] [--reps 4] [--out DIR]

The workload is bench.py's: B = 1, fp16 mode, synthetic weights and frames, `--windows` distinct windows per step, the
module's CUDA-graph path, warmed up as bench.py does.  Two runs in one process:
  timed    `--reps` steps with CUDA events around each window, profiler off: the event-timed ms per window.
  traced   one step under torch.profiler (CUDA activity); the Chrome trace goes to DIR/window_trace.pt.trace.json and
           every kernel in it is attributed to a layer.
Attribution follows the fixed launch order of one backbone stage: pack, SFENet1, SFENet2, 12 x (3 growth convs + fused
tail), GFF.0, GFF.1, UPNet.0, UPNet.2.  SFENet2 and GFF.1 run the same kernel instantiation, so layers are told apart by
their position after the stage's pack kernel, not by name.  `convlstm_kernel` launches are the ConvLSTM cells.

Each layer's floor is computed from the window's shapes (layer_work below): its FLOPs over the dense fp16 tensor rate
(989 TFLOP/s, the H100 SXM data sheet; the ConvLSTM runs fp32 FMAs on the CUDA cores, 67 TFLOP/s) or its bytes over
3.35 TB/s of HBM3, whichever is larger; the table names the bound.  Those rates are for a card allowed 700 W, so the
card's name, power limit and SM clock are read in the same run and printed beside the table.

Without a CUDA device the script prints the floor table and stops with an error: there is no CPU timing."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TENSOR_FLOPS = 989e12        # dense fp16, H100 SXM data sheet
FP32_FLOPS = 67e12           # fp32 CUDA cores, same
HBM_BYTES = 3.35e12          # HBM3, same

G0, G, D, CGROW = 96, 32, 12, 4
STAGES = ((5, 2), (6, 3), (4, 5), (2, 5))     # (backbone calls, frames per call) of the four stages, in launch order
LSTM_CELLS = (3, 2, 1)                        # cells per ConvLSTM launch (before stages 1, 2, 3)
STAGE_LAYERS = (["SFENet1", "SFENet2"] + ["RDB growth convs", "RDB growth convs", "RDB growth convs", "RDB tail"] * D
                + ["GFF.0", "GFF.1", "UPNet.0", "UPNet.2"])
ORDER = ["pack", "SFENet1", "SFENet2", "RDB growth convs", "RDB tail", "GFF.0", "GFF.1", "UPNet.0", "UPNet.2", "ConvLSTM"]


def align32(c):
    return (c + 31) // 32 * 32


def layer_work(H, W):
    """{layer: [fp16 tensor FLOPs, fp32 FLOPs, HBM bytes, launches]} of one full window at H x W (B = 1).  Bytes count
    each tensor a layer must read or write once: activations fp16, frames and outputs fp32."""
    h, w = H // 2, W // 2
    work = {k: [0.0, 0.0, 0.0, 0] for k in ORDER}

    def add(k, tflop=0.0, fflop=0.0, nbytes=0.0, launches=1):
        e = work[k]
        e[0] += tflop; e[1] += fflop; e[2] += nbytes; e[3] += launches

    for n, nf in STAGES:
        P, Q = n * h * w, n * H * W                   # low-res and full-res positions of the stage
        cin1 = 12 * nf                                # pixel-reshuffled frames (RDN.py:211)
        add("pack", nbytes=Q * nf * 3 * 4 + P * align32(cin1) * 2)
        add("SFENet1", 2 * P * G0 * cin1 * 25, nbytes=P * (align32(cin1) + G0) * 2)
        add("SFENet2", 2 * P * G0 * G0 * 9, nbytes=P * 2 * G0 * 2)
        for _ in range(D):
            for c in range(CGROW - 1):
                add("RDB growth convs", 2 * P * G * (G0 + c * G) * 9, nbytes=P * (G0 + c * G + G) * 2)
            cin3 = G0 + (CGROW - 1) * G
            add("RDB tail", 2 * P * (G * cin3 * 9 + G0 * (G0 + CGROW * G)), nbytes=P * (cin3 + G0) * 2)
        add("GFF.0", 2 * P * G0 * D * G0, nbytes=P * (D * G0 + G0) * 2)
        add("GFF.1", 2 * P * G0 * G0 * 9, nbytes=P * 3 * G0 * 2)
        add("UPNet.0", 2 * P * 4 * 64 * G0 * 9, nbytes=P * (G0 + 4 * 64) * 2)
        add("UPNet.2", 2 * Q * 3 * 64 * 9, nbytes=Q * (64 * 2 + nf * 3 * 4 + 3 * 4))
    for cells in LSTM_CELLS:
        add("ConvLSTM", fflop=cells * 2 * H * W * 12 * 3 * 9, nbytes=cells * H * W * 3 * 4 * 2)
    return work


def floor_ms(e):
    t_tc, t_fp, t_mem = e[0] / TENSOR_FLOPS, e[1] / FP32_FLOPS, e[2] / HBM_BYTES
    t = max(t_tc, t_fp, t_mem)
    bound = "HBM" if t == t_mem else ("fp16 TC" if t == t_tc else "fp32 FMA")
    return t * 1e3, bound


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.sw_power_cap"
    try:
        import torch
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        name, power, sm, sm_max, cap = [s.strip() for s in r.stdout.strip().split(",")]
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}
    return {"name": name, "power_limit": power, "sm_clock": sm, "max_sm_clock": sm_max, "sw_power_cap": cap}


def attribute(kernels):
    """kernels: [(name, start_us, dur_us)] in start order -> ([(layer, dur_us)], number of stages seen).  A stage starts
    at its pack kernel; every conv or tail launch after it takes the next position of STAGE_LAYERS."""
    out, pos, stages = [], None, 0
    for name, _, dur in kernels:
        if "pack_frames_kernel" in name:
            pos, stages = 0, stages + 1
            out.append(("pack", dur))
        elif "convlstm_kernel" in name:
            out.append(("ConvLSTM", dur))
        elif "conv_igemm_kernel" in name or "rdb_tail_kernel" in name:
            if pos is None or pos >= len(STAGE_LAYERS):
                raise SystemExit(f"profile_window: conv launch outside a stage's launch order: {name}")
            layer = STAGE_LAYERS[pos]
            if (layer == "RDB tail") != ("rdb_tail_kernel" in name):
                raise SystemExit(f"profile_window: launch {pos} of a stage is {name}, expected {layer}")
            out.append((layer, dur))
            pos += 1
        else:
            out.append(("other", dur))
    return out, stages


def print_floors(work):
    print(f"{'layer':<18}{'launches':>9}{'GFLOP':>10}{'MB':>10}{'floor ms':>10}  bound")
    for k in ORDER:
        e = work[k]
        f, bound = floor_ms(e)
        print(f"{k:<18}{e[3]:>9}{(e[0] + e[1]) / 1e9:>10.1f}{e[2] / 1e6:>10.1f}{f:>10.3f}  {bound}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--windows", type=int, default=5, help="distinct windows per step (bench.py: 5)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=4, help="event-timed steps")
    ap.add_argument("--out", default="profile_window_out")
    args = ap.parse_args()
    H, W, S = args.height, args.width, args.windows
    work = layer_work(H, W)
    print(f"window {H}x{W}, B = 1: per-window work and floors (fp16 TC {TENSOR_FLOPS / 1e12:.0f} TFLOP/s, "
          f"fp32 {FP32_FLOPS / 1e12:.0f} TFLOP/s, HBM {HBM_BYTES / 1e12:.2f} TB/s)")
    print_floors(work)

    import torch
    if not torch.cuda.is_available():
        sys.exit("profile_window: needs a CUDA device for the timed and traced runs (there is no CPU timing)")
    from bin_b200 import _lib, rdn
    from oracle import bin_oracle as O
    _lib.check(_lib.lib().bin_check_device())
    os.makedirs(args.out, exist_ok=True)
    res = {"H": H, "W": W, "windows_per_step": S, "card_before": card()}
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    net = net.cuda().eval()
    wins = [[f.cuda() for f in O.synth_frames(6, 1, H, W, seed=1234 + i, smooth=True)] for i in range(S)]
    with torch.no_grad():
        outs = None
        for _ in range(args.warmup):
            for w_ in wins:
                outs = net(*w_)
        torch.cuda.synchronize()
        # ---- timed: CUDA events around every window, profiler off
        ev = [[torch.cuda.Event(enable_timing=True) for _ in range(S + 1)] for _ in range(args.reps)]
        for r in range(args.reps):
            ev[r][0].record()
            for i, w_ in enumerate(wins):
                outs = net(*w_)
                ev[r][i + 1].record()
        torch.cuda.synchronize()
        per_window = [ev[r][i].elapsed_time(ev[r][i + 1]) for r in range(args.reps) for i in range(S)]
        res["event_ms_per_window"] = {"median": statistics.median(per_window), "min": min(per_window), "max": max(per_window),
                                      "mean_of_steps": sum(ev[r][0].elapsed_time(ev[r][S]) for r in range(args.reps)) / (args.reps * S)}
        # ---- traced: one step under the profiler, in a run of its own
        from torch.profiler import ProfilerActivity, profile
        trace = os.path.join(args.out, "window_trace.pt.trace.json")
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for w_ in wins:
                outs = net(*w_)
            torch.cuda.synchronize()
        prof.export_chrome_trace(trace)
        del outs
    res["card_after"] = card()
    with open(trace) as fh:
        events = json.load(fh)["traceEvents"]
    kernels = sorted(((e["name"], float(e["ts"]), float(e["dur"])) for e in events
                      if e.get("ph") == "X" and e.get("cat") == "kernel"), key=lambda k: k[1])
    if not kernels:
        sys.exit("profile_window: the trace holds no kernel events")
    attributed, stages = attribute(kernels)
    if stages != 4 * S:
        sys.exit(f"profile_window: traced {stages} backbone stages, expected {4 * S}")
    gaps = sum(max(0.0, b[1] - (a[1] + a[2])) for a, b in zip(kernels, kernels[1:]))
    span = kernels[-1][1] + kernels[-1][2] - kernels[0][1]
    per = {}
    for layer, dur in attributed:
        p = per.setdefault(layer, [0.0, 0])
        p[0] += dur / 1e3 / S
        p[1] += 1
    total = sum(p[0] for p in per.values())
    floor_total = 0.0
    rows = []
    print(f"\ntraced: {len(kernels)} kernels over {S} windows; ms per window")
    print(f"{'layer':<18}{'ms':>9}{'share':>8}{'launches':>9}{'floor ms':>10}{'x floor':>9}  bound")
    for k in ORDER + ["other"]:
        if k not in per:
            continue
        ms, n = per[k]
        f, bound = floor_ms(work[k]) if k in work else (0.0, "-")
        floor_total += f
        rows.append({"layer": k, "ms_per_window": ms, "launches_per_window": n / S, "floor_ms": f, "bound": bound})
        ratio = f"{ms / f:>9.2f}" if f > 0 else f"{'-':>9}"
        print(f"{k:<18}{ms:>9.3f}{ms / total:>8.1%}{n / S:>9.0f}{f:>10.3f}{ratio}  {bound}")
    ewin = res["event_ms_per_window"]["median"]
    print(f"{'kernel sum':<18}{total:>9.3f}{'':>8}{len(kernels) / S:>9.0f}{floor_total:>10.3f}{total / floor_total:>9.2f}")
    print(f"event-timed window (median of {args.reps * S}, profiler off): {ewin:.3f} ms; kernel sum / window = "
          f"{total / ewin:.3f}; traced gaps between kernels {gaps / 1e3 / S:.3f} ms per window "
          f"(traced span {span / 1e3 / S:.3f} ms per window)")
    for tag in ("card_before", "card_after"):
        print(f"{tag}: {res[tag]}")
    res.update({"layers": rows, "kernel_sum_ms_per_window": total, "gap_ms_per_window": gaps / 1e3 / S,
                "traced_span_ms_per_window": span / 1e3 / S, "trace": trace})
    with open(os.path.join(args.out, "profile_window.json"), "w") as fh:
        fh.write(json.dumps(res) + "\n")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
