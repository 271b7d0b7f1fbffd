"""Time the evaluation metrics (bin_b200.metrics) on one 720x1280x3 uint8 pair -- the frame test.py scores four times
per window -- and print the card, the CPU time of the fp64 oracle restatements on the same pair, and the least time
the hardware could take (fp64 operations and bytes the kernel needs, counted from the shape).

    python tools/bench_metrics.py [--iters 50] [--warmup 5]

Cases (CUDA events, after warm-up):
  kernel        back-to-back bin_image_metrics_u8 launches on device-resident images, no host synchronisation;
  device        image_metrics() on device-resident tensors (launch + the 32-byte result copy + synchronisation);
  numpy         image_metrics() on numpy arrays (adds the two uploads the skimage / util drop-ins do);
  test.py pair  compare_psnr(res, gt) + compare_ssim(res, gt, multichannel=True) on numpy arrays (two calls).
Needs a CUDA device; there is no CPU fallback."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bin_b200 import _lib, metrics             # noqa: E402
from bin_b200.rdn import _workspace            # noqa: E402
from oracle import metrics_oracle as M         # noqa: E402

H, W, CH = 720, 1280, 3
# per (pixel, channel): Gaussian horizontal + vertical passes, 5 quantities x 11 taps x 2 flops each, plus the two
# SSIM formulas (~15 fp64 operations each).  The box sums are int32.  Inputs are read once.
FP64_OPS_PER_PX = 2 * 5 * 11 * 2 + 2 * 15
H100_FP64_TFLOPS = 34.0          # H100 SXM data sheet, FP64 (non-tensor) at 700 W
H100_HBM_TBPS = 3.35


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [s.strip() for s in r.stdout.strip().split(",")]
    except Exception as e:  # noqa: BLE001
        name, power, clock = torch.cuda.get_device_name(), f"unknown ({e})", "unknown"
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def timed_ms(fn, iters, warm):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_metrics: needs a CUDA device (the metrics have no CPU path)")
    iters = max(args.iters, 50)
    rng = np.random.default_rng(0)
    from scipy.ndimage import gaussian_filter
    z = gaussian_filter(rng.standard_normal((H, W, CH)), sigma=(4.0, 4.0, 0.0))
    a = np.clip(np.round((z - z.min()) / (z.max() - z.min()) * 235 + 10), 0, 255).astype(np.uint8)
    b = np.clip(a.astype(np.int32) + rng.normal(0, 4, size=a.shape).round().astype(np.int32), 0, 255).astype(np.uint8)
    ta, tb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()

    L = _lib.lib()
    _lib.check(L.bin_check_device())
    ws = _workspace(ta.device, L.bin_image_metrics_workspace_bytes(H, W))
    out4 = torch.empty(4, dtype=torch.float64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    launch = lambda: _lib.check(L.bin_image_metrics_u8(ta.data_ptr(), tb.data_ptr(), H, W, CH, out4.data_ptr(),  # noqa: E731
                                                       ws.data_ptr(), ws.numel(), st))
    res = {"card": card(), "shape": [H, W, CH], "iters": iters}
    res["kernel_ms"] = timed_ms(launch, iters, args.warmup)
    res["device_ms"] = timed_ms(lambda: metrics.image_metrics(ta, tb), iters, args.warmup)
    res["numpy_ms"] = timed_ms(lambda: metrics.image_metrics(a, b), iters, args.warmup)
    res["test_py_pair_ms"] = timed_ms(lambda: (metrics.compare_psnr(a, b), metrics.compare_ssim(a, b, multichannel=True)),
                                      iters, args.warmup)

    gpu = metrics.image_metrics(ta, tb)
    cpu = {}
    for name, fn in (("ssim_gauss11", M.ssim_gauss11), ("ssim_box7", M.ssim_box7), ("psnr", M.psnr)):
        t0 = time.perf_counter()
        v = fn(a, b)
        cpu[name + "_ms"] = (time.perf_counter() - t0) * 1e3
        cpu[name] = v
    res["cpu_oracle"] = dict(cpu, cores=os.cpu_count())
    res["gpu_values"] = {"mean_abs": gpu[0], "mse": gpu[1], "ssim_gauss11": gpu[2], "ssim_box7": gpu[3]}
    res["max_abs_diff_vs_oracle"] = max(abs(gpu[2] - cpu["ssim_gauss11"]), abs(gpu[3] - cpu["ssim_box7"]))

    n = H * W * CH
    flops, nbytes = n * FP64_OPS_PER_PX, 2 * n
    t_flop, t_byte = flops / (H100_FP64_TFLOPS * 1e12) * 1e3, nbytes / (H100_HBM_TBPS * 1e12) * 1e3
    res["bound"] = {"fp64_ops": flops, "bytes": nbytes, "fp64_ms_at_datasheet_peak": t_flop,
                    "hbm_ms_at_datasheet_peak": t_byte, "bound_by": "fp64" if t_flop > t_byte else "hbm",
                    "kernel_share_of_bound": max(t_flop, t_byte) / res["kernel_ms"]}
    c = res["card"]
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}")
    print(f"720x1280x3 pair, {iters} calls: kernel {res['kernel_ms'] * 1e3:.1f} us | image_metrics device-resident "
          f"{res['device_ms'] * 1e3:.1f} us | from numpy {res['numpy_ms'] * 1e3:.1f} us | test.py psnr+ssim pair "
          f"{res['test_py_pair_ms'] * 1e3:.1f} us")
    print(f"CPU oracle ({os.cpu_count()} cores): gauss11 {cpu['ssim_gauss11_ms']:.1f} ms, box7 {cpu['ssim_box7_ms']:.1f} ms, "
          f"psnr {cpu['psnr_ms']:.1f} ms; max |GPU - oracle| SSIM {res['max_abs_diff_vs_oracle']:.2e}")
    bd = res["bound"]
    print(f"bound: {flops / 1e6:.0f} MFLOP fp64 -> {t_flop * 1e3:.1f} us, {nbytes / 1e6:.1f} MB -> {t_byte * 1e3:.1f} us "
          f"({bd['bound_by']}-bound); kernel reaches {bd['kernel_share_of_bound']:.0%} of it")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
