"""Time the x4 flip self-ensemble (rdn.set_self_ensemble(net, "flipx4")) against the plain window and against the same
ensemble built from four sequential plain calls with torch flips, and time its two kernels alone.  Prints the card, its
power limit and SM clocks, read in the same run.

    python tools/bench_ensemble.py [--reps 10] [--warmup 2] [--sizes 768x1344,720x1280]

Per size (H x W, B = 1, fp16 mode, synthetic weights and frames):
  plain        one window through the module (its CUDA-graph path), CUDA events, median of --reps;
  ensemble     one ensemble call (expand, one window at batch 4B, mean), median of --reps;
  sequential   four plain calls on torch.flip'ped frames, the outputs flipped back, summed and divided by 4 in torch:
               what utils/test_util.py:110-132 does; timed alternately with the ensemble in the same loop;
  kernels      bin_flipx4_expand over the 6 frames and bin_flipx4_mean over the 14 outputs, 50 back-to-back launches
               each on preallocated tensors; GB/s = bytes each must move / kernel time, against 3.35 TB/s;
  memory       torch.cuda.max_memory_allocated() growth of one ensemble call with no cached workspace, beside the
               workspace of the window's largest stage at 4B (bin_backbone_workspace_bytes_p) + the frame, intermediate
               and output tensors it needs.
Needs a CUDA device; there is no CPU fallback."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bin_b200 import _lib, rdn                 # noqa: E402
from oracle import bin_oracle as O             # noqa: E402

H100_HBM_TBPS = 3.35
ORIENTATIONS = [None, (-1,), (-2,), (-2, -1)]


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


def sequential(net, frames):
    acc = None
    for dims in ORIENTATIONS:
        outs = net(*[f if dims is None else torch.flip(f, dims) for f in frames])
        outs = [o if dims is None else torch.flip(o, dims) for o in outs]
        acc = outs if acc is None else [a + o for a, o in zip(acc, outs)]
    return [a / 4 for a in acc]


def kernel_ms(fn_name, srcs, dsts, B, H, W, iters=50):
    L = _lib.lib()
    fn = getattr(L, fn_name)
    sp = (C.c_void_p * len(srcs))(*[t.data_ptr() for t in srcs])
    dp = (C.c_void_p * len(dsts))(*[t.data_ptr() for t in dsts])
    st = torch.cuda.current_stream().cuda_stream
    launch = lambda: _lib.check(fn(sp, dp, len(srcs), B, H, W, st))      # noqa: E731
    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    return event_ms(lambda: [launch() for _ in range(iters)]) / iters


def run_size(net, H, W, reps, warmup):
    B = 1
    frames = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=3, smooth=True)]
    plane = B * 3 * H * W * 4                                   # bytes of one (B,3,H,W) fp32 tensor
    res = {"H": H, "W": W, "B": B, "precision": "fp16"}
    with torch.no_grad():
        # memory of one ensemble call, from a state with no cached workspace and no captured graph
        net.__dict__.pop("_graph_entry", None)
        rdn.release_workspaces()
        torch.cuda.empty_cache()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        rdn.set_self_ensemble(net, "flipx4")
        outs = net(*frames)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        del outs
        # (frames per call, calls) of the window's four stages; 9 intermediate images (6 ConvLSTM h, 3 step-1 outputs)
        ws = max(_lib.lib().bin_backbone_workspace_bytes_p(nf, n * 4 * B, H, W, 0) for nf, n in ((2, 5), (3, 6), (5, 4), (5, 2)))
        tensors = (6 * 4 + 14 * 4 + 9 * 4 + 14) * plane        # expanded frames, 4B outputs and intermediates, the 14 means
        res["memory"] = {"peak_growth_bytes": peak, "stage_workspace_4B_bytes": ws, "tensor_bytes": tensors,
                         "peak_over_expected": peak / (ws + tensors)}

        ens = lambda: net(*frames)                              # noqa: E731
        for _ in range(warmup):
            ens()
        rdn.set_self_ensemble(net, None)
        for _ in range(warmup):
            net(*frames)
            sequential(net, frames)
        torch.cuda.synchronize()
        plain_t, ens_t, seq_t = [], [], []
        for _ in range(reps):
            plain_t.append(event_ms(lambda: net(*frames)))
            seq_t.append(event_ms(lambda: sequential(net, frames)))
            rdn.set_self_ensemble(net, "flipx4")
            ens_t.append(event_ms(ens))
            rdn.set_self_ensemble(net, None)
        res["plain_ms"] = statistics.median(plain_t)
        res["ensemble_ms"] = statistics.median(ens_t)
        res["sequential_ms"] = statistics.median(seq_t)
        res["ensemble_over_sequential"] = res["ensemble_ms"] / res["sequential_ms"]
        res["ensemble_over_plain"] = res["ensemble_ms"] / res["plain_ms"]
        res["spread_ms"] = {"plain": [min(plain_t), max(plain_t)], "ensemble": [min(ens_t), max(ens_t)],
                            "sequential": [min(seq_t), max(seq_t)]}

        big = [torch.empty((4 * B, 3, H, W), device="cuda") for _ in range(14)]
        small = [torch.empty((B, 3, H, W), device="cuda") for _ in range(14)]
        kx = kernel_ms("bin_flipx4_expand", frames, big[:6], B, H, W)
        km = kernel_ms("bin_flipx4_mean", big, small, B, H, W)
        bx, bm = 6 * 5 * plane, 14 * 5 * plane                  # read 1 + write 4 / read 4 + write 1 tensors per entry
        res["kernels"] = {
            "expand_ms": kx, "expand_bytes": bx, "expand_GBps": bx / kx / 1e6, "expand_share_of_hbm_peak": bx / kx / 1e9 / H100_HBM_TBPS,
            "mean_ms": km, "mean_bytes": bm, "mean_GBps": bm / km / 1e6, "mean_share_of_hbm_peak": bm / km / 1e9 / H100_HBM_TBPS,
            "share_of_ensemble": (kx + km) / res["ensemble_ms"]}
        del big, small
    net.__dict__.pop("_graph_entry", None)
    rdn.release_workspaces()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sizes", default="768x1344,720x1280")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ensemble: needs a CUDA device (the ensemble has no CPU path)")
    _lib.check(_lib.lib().bin_check_device())
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    net = net.cuda().eval()
    out = {"card_before": card(), "sizes": []}
    for s in args.sizes.split(","):
        H, W = (int(v) for v in s.split("x"))
        r = run_size(net, H, W, args.reps, args.warmup)
        out["sizes"].append(r)
        k, m = r["kernels"], r["memory"]
        print(f"{H}x{W} B=1 fp16: plain {r['plain_ms']:.1f} ms | ensemble {r['ensemble_ms']:.1f} ms | 4 sequential calls + "
              f"torch flips {r['sequential_ms']:.1f} ms (ensemble / sequential {r['ensemble_over_sequential']:.3f})")
        print(f"  expand {k['expand_ms'] * 1e3:.0f} us ({k['expand_GBps']:.0f} GB/s, {k['expand_share_of_hbm_peak']:.0%} of 3.35 TB/s)"
              f" | mean {k['mean_ms'] * 1e3:.0f} us ({k['mean_GBps']:.0f} GB/s, {k['mean_share_of_hbm_peak']:.0%}) | both "
              f"{k['share_of_ensemble']:.2%} of the ensemble")
        print(f"  peak memory growth {m['peak_growth_bytes'] / 1e9:.2f} GB vs stage workspace {m['stage_workspace_4B_bytes'] / 1e9:.2f}"
              f" GB + tensors {m['tensor_bytes'] / 1e9:.2f} GB (ratio {m['peak_over_expected']:.3f})")
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
