"""Time a window that computes only the outputs test.py writes (rdn.set_outputs(net, (13, 8, 12))) against the full
14-output window, through the module and through StreamingBIN.  Prints the card, its power limit and SM clocks, read in
the same run.

    python tools/bench_outputs.py [--reps 10] [--rounds 2] [--warmup 3] [--sizes 720x1280,768x1344]

Per size (H x W, B = 1, fp16 mode, synthetic weights and frames):
  window     one call of the module on its CUDA-graph path: 17 backbone calls for the full window, 13 with the
             selection.  The two variants alternate inside one loop (one net each, so that both keep their captured
             graph); CUDA events around each call; median over --rounds x --reps.
  streamed   one StreamingBIN.push in steady state: 13 backbone calls for the full window, 10 with the selection.  The
             two streams alternate frame by frame over the same synthetic video.
  memory     torch.cuda.max_memory_allocated() growth of one eager window call from a state with no cached workspace,
             and of one steady-state push.  The window workspace is sized for the full window either way; the
             selection saves output tensors only.
  expected   the ratio of backbone calls (13/17, 10/13), which is what the time ratio would be if every stage used the
             card equally well at its smaller batch.
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
from bin_b200 import _lib, rdn                 # noqa: E402
from bin_b200.streaming import StreamingBIN    # noqa: E402
from oracle import bin_oracle as O             # noqa: E402

WANTED = (13, 8, 12)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        name, power, sm, sm_max = [s.strip() for s in r.stdout.strip().split(",")]
    except Exception as e:  # noqa: BLE001
        name, power, sm, sm_max = torch.cuda.get_device_name(), f"unknown ({e})", "unknown", "unknown"
    return {"name": name, "power_limit": power, "sm_clock": sm, "max_sm_clock": sm_max}


def event_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def peak_growth(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del out
    return peak


def summary(full, sel, expected):
    return {"full_ms": statistics.median(full), "selected_ms": statistics.median(sel),
            "ratio": statistics.median(sel) / statistics.median(full), "expected_ratio_from_calls": expected,
            "spread_ms": {"full": [min(full), max(full)], "selected": [min(sel), max(sel)]}}


def run_size(nets, H, W, reps, rounds, warmup):
    full_net, sel_net = nets
    frames = [f.cuda() for f in O.synth_frames(6, 1, H, W, seed=3, smooth=True)]
    res = {"H": H, "W": W, "B": 1, "precision": "fp16", "wanted": list(WANTED)}
    with torch.no_grad():
        # memory of one eager call per variant, from a state with no cached workspace and no captured graph
        os.environ["BIN_B200_GRAPH"] = "0"
        mem = {}
        for tag, net in (("full", full_net), ("selected", sel_net)):
            rdn.release_workspaces()
            torch.cuda.empty_cache()
            mem[tag + "_window_peak_bytes"] = peak_growth(lambda: net(*frames))
        os.environ["BIN_B200_GRAPH"] = "1"
        rdn.release_workspaces()
        torch.cuda.empty_cache()

        # ---- module window, graphed path, the variants alternating
        for _ in range(warmup):
            full_net(*frames)
            sel_net(*frames)
        torch.cuda.synchronize()
        full_t, sel_t = [], []
        for _ in range(rounds):
            for _ in range(reps):
                full_t.append(event_ms(lambda: full_net(*frames)))
                sel_t.append(event_ms(lambda: sel_net(*frames)))
        res["window"] = summary(full_t, sel_t, 13 / 17)
        for net in nets:
            net.__dict__.pop("_graph_entry", None)
        torch.cuda.empty_cache()

        # ---- streaming, steady state, the two streams alternating frame by frame over one video
        first_timed = 6 + warmup                                # pushes 0..4 fill the window, push 5 is the first window
        n = first_timed + rounds * reps
        video = [f.cuda() for f in O.synth_frames(8, 1, H, W, seed=5, smooth=True)]
        streams = (StreamingBIN(full_net), StreamingBIN(sel_net))
        full_t, sel_t = [], []
        for k in range(n):
            f = video[k % len(video)]
            for tag, st, times in zip(("full", "selected"), streams, (full_t, sel_t)):
                if k == first_timed - 1:
                    mem[tag + "_stream_push_peak_bytes"] = peak_growth(lambda: st.push(f))
                elif k >= first_timed:
                    times.append(event_ms(lambda: st.push(f)))
                else:
                    st.push(f)
        res["streamed"] = summary(full_t, sel_t, 10 / 13)
        res["streamed"]["backbone_calls"] = {"full": streams[0].backbone_calls, "selected": streams[1].backbone_calls,
                                             "windows": n - 5}
        res["memory"] = mem
        for st in streams:
            st.reset()
    rdn.release_workspaces()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sizes", default="720x1280,768x1344")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_outputs: needs a CUDA device (the window has no CPU path)")
    _lib.check(_lib.lib().bin_check_device())
    nets = []
    for wanted in (None, WANTED):
        net = rdn.bin_stage4_lstm()
        net.load_state_dict(O.synth_state_dict(0), strict=True)
        nets.append(rdn.set_outputs(net.cuda().eval(), wanted))
    out = {"card_before": card(), "sizes": []}
    for s in args.sizes.split(","):
        H, W = (int(v) for v in s.split("x"))
        r = run_size(nets, H, W, args.reps, args.rounds, args.warmup)
        out["sizes"].append(r)
        w, st, m = r["window"], r["streamed"], r["memory"]
        print(f"{H}x{W} B=1 fp16: window full {w['full_ms']:.1f} ms | {WANTED} {w['selected_ms']:.1f} ms | ratio {w['ratio']:.3f} "
              f"(calls 13/17 = {13 / 17:.3f})")
        print(f"  streamed window full {st['full_ms']:.1f} ms | {WANTED} {st['selected_ms']:.1f} ms | ratio {st['ratio']:.3f} "
              f"(calls 10/13 = {10 / 13:.3f})")
        print(f"  spread window {w['spread_ms']} streamed {st['spread_ms']}")
        print("  peak memory growth, GB: " + ", ".join(f"{k[:-len('_peak_bytes')]} {v / 1e9:.3f}" for k, v in m.items()))
    out["card_after"] = card()
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
