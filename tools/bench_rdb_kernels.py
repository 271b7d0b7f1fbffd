"""Time the residual dense block's kernels alone at the window's shapes: the three x-stacked growth convs
(conv_igemm_kernel<32, 3, P8, SX>) as one launch set, and the fused tail (rdb_tail_kernel<96>).

    python tools/bench_rdb_kernels.py [--batch 5] [--height 360] [--width 640] [--launches 50] [--reps 5]

Shapes and plane layouts are those of run_rdb for an inner block of the shipped backbone (G0 = 96, D = 12) in one
backbone stage of bench.py's window: x is G0 planes of the D*G0-channel concat, the growth maps are a 16-plane tensor
(conv c reads x and growth planes [0, 4c) and writes planes [4c, 4c + 4)), the tail writes the next G0 planes of the
concat.  Each figure is the minimum over --reps runs of --launches back-to-back launch sets between two CUDA events.

Work is what the algorithm needs: every input and output byte once, 2 FLOPs per MAC.  Fractions are of the H100 SXM
data sheet (3.35 TB/s HBM3, 989 TFLOP/s dense fp16), which assumes a 700 W card; the card's name, power limit and SM
clock are read in the same run and printed beside the numbers."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from profile_window import HBM_BYTES, TENSOR_FLOPS, card  # noqa: E402

G0, G, D, P = 96, 32, 12, 12        # P = G0 / 8 planes


def work(B, H, W):
    """{kernel set: (FLOPs, bytes)} per launch set."""
    n = B * H * W
    grow_f = sum(2 * n * G * (G0 + c * G) * 9 for c in range(3))
    grow_b = sum(n * (G0 + c * G + G) * 2 for c in range(3))
    cin3 = G0 + 3 * G
    tail_f = 2 * n * (G * cin3 * 9 + G0 * (cin3 + G))
    tail_b = n * (cin3 + G0) * 2
    return {"growth convs": (grow_f, grow_b), "tail": (tail_f, tail_b)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=5)
    ap.add_argument("--height", type=int, default=360)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--launches", type=int, default=50, help="launch sets between two events")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    B, H, W = args.batch, args.height, args.width

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_rdb_kernels: needs a CUDA device (there is no CPU timing)")
    from bin_b200 import _lib, ops
    _lib.check(_lib.lib().bin_check_device())
    dev = "cuda"
    gen = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *sh: torch.randn(*sh, device=dev, generator=gen)
    cat = rnd(B, P * D, H, W, 8).half()            # x = planes [0, P), the tail writes planes [P, 2P)
    g = torch.zeros(B, 16, H, W, 8, device=dev).half()
    grow = []
    for c in range(3):
        cin = G0 + c * G
        w = rnd(G, cin, 3, 3) / (cin * 9) ** 0.5
        grow.append((ops.pack_conv_weight(w, G, cin), ops.pad_bias(rnd(G) * 0.1, G), c))
    w3, wl = rnd(G, G0 + 3 * G, 3, 3) / ((G0 + 3 * G) * 9) ** 0.5, rnd(G0, G0 + 4 * G, 1, 1) / (G0 + 4 * G) ** 0.5
    p3, b3 = ops.pack_conv_weight(w3, G, G0 + 3 * G), ops.pad_bias(rnd(G) * 0.1, G)
    pl, bl = ops.pack_conv_weight(wl, G0, G0 + 4 * G), ops.pad_bias(rnd(G0) * 0.1, G0)

    def growth():
        for wp, bp, c in grow:
            ops.conv_fwd(cat, wp, bp, 3, G, in0_planes=P, in1=g, in1_planes=4 * c, relu=True, out=g, out_plane0=4 * c)

    def tail():
        ops.rdb_tail_fwd(cat, g, p3, b3, pl, bl, cat, x_plane0=0, g_plane0=0, out_plane0=P)

    res = {"B": B, "H": H, "W": W, "launches": args.launches, "reps": args.reps, "card_before": card()}
    for name, fn in (("growth convs", growth), ("tail", tail)):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.launches):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / args.launches)
        ms = min(ts)
        flops, nbytes = work(B, H, W)[name]
        t_tc, t_mem = flops / TENSOR_FLOPS * 1e3, nbytes / HBM_BYTES * 1e3
        res[name] = {"ms": ms, "ms_all_reps": ts, "GB_s": nbytes / ms / 1e6, "TFLOP_s": flops / ms / 1e9,
                     "frac_hbm": t_mem / ms, "frac_tensor": t_tc / ms, "floor_ms": max(t_tc, t_mem),
                     "bound": "HBM" if t_mem >= t_tc else "fp16 TC"}
        r = res[name]
        print(f"{name:<14}{ms:8.4f} ms  {r['GB_s']:7.0f} GB/s ({r['frac_hbm']:.1%} of HBM)  {r['TFLOP_s']:6.1f} TFLOP/s "
              f"({r['frac_tensor']:.1%} of fp16 TC)  floor {r['floor_ms']:.3f} ms ({r['bound']})", flush=True)
    res["card_after"] = card()
    print(f"card: {res['card_before']}\ncard after: {res['card_after']}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
