#!/usr/bin/env python
"""bench.py -- BIN hot path on H100: 720p frame-windows/sec (BASELINE.json metric).

One "step" = `--windows-per-step` (default 5) forwards of the shipped 6-frame bin_stage4 network (the path test.py
runs, SURVEY 8d config 2b) on independent synthetic 1280x720 windows per GPU; windows are independent, so N GPUs run
N x that many windows per step with no collective in the loop (weak scaling; one weight broadcast at start-up,
excluded from the timed region and timed separately).  Five windows per step make the timed region of the driver's
20-step run ~3 s, long enough that one slow rank shows up in the per-rank record instead of in the noise.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference|reference-cuda]
                    [--height H --width W] [--windows-per-step S] [--no-extras] [--dump-outputs DIR]

Prints ONE JSON line (rank 0).  `value` = device-resident windows/s, `e2e` = the same metric through the module call
with pinned-host inputs (6 frames H2D per window) and the 3 images test.py writes (outputs 13, 8, 12) copied back D2H
inside the timed region.  `--impl reference` times the reference's CPU PyTorch path (the unmodified reference when it
is present under baseline/_ref, else the line-cited oracle port) on REAL 1280x720 windows.
`--dump-outputs DIR` writes, after the timed steps, the 14 outputs of every window of the last timed step (recomputed
untimed from the same inputs and checked bit for bit against the last window's timed outputs) as
DIR/window<i>_out<k>.npy (float32; a fixed seeded sample of each flattened output when all of them would exceed 64 MB).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "720p frame-windows/sec"
UNIT = "windows/s"
MACS_PER_PX = 14_234_976          # SURVEY 8d: conv MACs per input pixel, reference-as-executed (20 backbone calls)
EXECUTED_FRACTION = (5 * 702_720 + 6 * 709_920 + 6 * 724_320 + 6 * 648) / MACS_PER_PX
# kernels per window: 4 batched backbone stages x (1 pack + 42 conv + 12 fused RDB tails) + 3 ConvLSTM launches (6 cells)
LAUNCHES_PER_WINDOW = 4 * (1 + 42 + 12) + 3


def peaks():
    # fallback = the H100 SXM data sheet (dense fp16/bf16, HBM3): peaks to divide by, not rates this code reaches
    p = {"bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0, "hbm_gbs": 3350.0, "source": "fallback"}
    try:
        d = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        p.update({k: d[k] for k in ("bf16_tflops", "bf16_tflops_sustained", "hbm_gbs") if k in d})
        p["source"] = "measured"
    except Exception:
        pass
    return p


class ClockSampler:
    """nvidia-smi clocks / throttle reasons of ONE GPU.  Every rank samples its own GPU.  The nvidia-smi process is started
    BEFORE the warm-up (NVML initialisation enumerates every GPU of the node and must not fall into the timed region: with
    one sampler per rank starting inside it, a 2-GPU run lost 20 %), polls at 5 Hz, and only the samples whose arrival time
    lies inside [mark_begin, mark_end] are used."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.idx, self.rows, self.proc = gpu_index, [], None
        self.t0 = self.t1 = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "200", "-i", str(self.idx)], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.time(), [c.strip() for c in line.split(",")]))

    def mark_begin(self):
        self.t0 = time.time()

    def mark_end(self):
        self.t1 = time.time()

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.25)
        self.proc.terminate()
        t0, t1 = self.t0 or 0.0, (self.t1 or time.time()) + 0.2
        rows = [r for (t, r) in self.rows if t0 <= t <= t1 and len(r) >= 8] or [r for (_, r) in self.rows if len(r) >= 8]
        sm = sorted(int(float(r[1])) for r in rows if r[1].replace(".", "").isdigit())
        reasons = set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in rows:
            for n, v in zip(names, r[4:8]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        mx = next((int(float(r[2])) for r in rows), None)
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_min_mhz": sm[0] if sm else None, "sm_max_mhz": mx,
                "reasons": sorted(reasons), "samples": len(sm)}


# ------------------------------------------------------------------------------------------------ CPU reference
def _reference_root():
    """The unmodified reference, when a copy of it is installed under baseline/_ref."""
    cand = os.path.join(ROOT, "baseline", "_ref")
    return cand if os.path.isfile(os.path.join(cand, "models", "archs", "RDN.py")) else None


def cpu_window_runner():
    """Returns (run(frames) -> outputs, kind): the reference's own bin_stage4_lstm on CPU when baseline/_ref is present -- kind "reference" -- else oracle/bin_oracle.py, the line-cited restatement that
    tests/golden pins to the reference's outputs -- kind "port".  Both are fp32 PyTorch CPU (oneDNN) graphs."""
    import torch
    from oracle import bin_oracle as O
    sd = O.synth_state_dict(0)
    root = _reference_root()
    if root is not None:
        try:
            sys.path.insert(0, root)
            import importlib
            R = importlib.import_module("models.archs.RDN")
            net = R.bin_stage4_lstm()
            net.load_state_dict(sd, strict=True)
            net.eval()

            def run(frames):
                with torch.no_grad():
                    return net(*frames)
            return run, "reference"
        except Exception:
            pass
        finally:
            if root in sys.path:
                sys.path.remove(root)

    def run_port(frames):
        with torch.no_grad():
            return O.window_forward(frames, sd)
    return run_port, "port"


def pick_cpu_threads(run, budget_s=20.0):
    """torch's CPU convolutions slow down when oversubscribed, so "all the host threads it can use" is found by a short
    sweep on a 192x320 window instead of assumed."""
    import torch
    from oracle import bin_oracle as O
    ncpu = os.cpu_count() or 1
    fr = O.synth_frames(6, 1, 192, 320, seed=1)
    best, sweep, t_start = None, {}, time.perf_counter()
    for th in [t for t in (8, 16, 32, 64) if t <= ncpu] or [ncpu]:
        torch.set_num_threads(th)
        run([f[:, :, :32, :32].contiguous() for f in fr])               # thread-pool / primitive warm-up
        t0 = time.perf_counter()
        run(fr)
        dt = time.perf_counter() - t0
        sweep[th] = round(dt, 3)
        if best is None or dt < best[1]:
            best = (th, dt)
        if time.perf_counter() - t_start > budget_s or dt > 1.3 * best[1]:      # past the sweet spot: more threads only hurt
            break
    torch.set_num_threads(best[0])
    return best[0], sweep


def run_reference(args):
    """`--impl reference`: the reference's own CPU implementation of the path, timed on REAL HxW (1280x720) windows.
    A full window costs ~1.5 minutes of CPU, so at most 1 (quarter-size) warm-up + 2 timed full windows are run whatever K / W ask for
    (`steps` in the line is what was actually timed; `requested_steps` what was asked)."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    import torch
    from oracle import bin_oracle as O
    H, W = args.height, args.width
    run, kind = cpu_window_runner()
    threads, sweep = pick_cpu_threads(run)
    fr = O.synth_frames(6, 1, H, W, seed=1234, smooth=True)
    nwarm = 1 if args.warmup >= 1 else 0
    nsteps = max(1, min(args.steps, 2))
    for _ in range(nwarm):                                   # thread pool / allocator warm-up on a quarter-size window (the
        run([f[:, :, :H // 4, :W // 4].contiguous() for f in fr])   # timed windows are full size; a full-size warm-up costs 1.5 min)
    ts = []
    for _ in range(nsteps):
        t0 = time.perf_counter()
        out = run(fr)
        ts.append(time.perf_counter() - t0)
    dt = sum(ts) / len(ts)
    val = 1.0 / dt
    cpu_model = ""
    try:
        cpu_model = next(l.split(":", 1)[1].strip() for l in open("/proc/cpuinfo") if l.startswith("model name"))
    except Exception:
        pass
    line = {"impl": "reference", "metric": METRIC, "value": val, "unit": UNIT, "n_gpus": args.gpus, "steps": nsteps,
            "requested_steps": args.steps, "warmup": nwarm, "ms_per_step": dt * 1e3, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": f"bin_stage4 6-frame window {W}x{H} (SURVEY 8d config 2b; what test.py runs)",
                       "frames": 6, "windows_per_gpu_per_step": 1, "outputs": 14,
                       "calls": "all 20 backbone calls + 12 ConvLSTM calls as the reference executes them"},
            "cpu_baseline": {"value": val, "unit": UNIT, "cores": threads, "kind": kind,
                             "host_cores": os.cpu_count(), "cpu_model": cpu_model, "torch": torch.__version__,
                             "thread_sweep_192x320_s": sweep,
                             "sample": f"{nsteps} full {W}x{H} 6-frame windows after {nwarm} quarter-size warm-up, {dt:.1f} s each "
                                       f"(per-window times {[round(t, 2) for t in ts]}); no pixel-count extrapolation"},
            "e2e": {"value": val, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "outputs_finite": bool(all(torch.isfinite(o).all() for o in out))}
    print(json.dumps(line), flush=True)


def eager_cuda_numbers(torch, dev, H, W, steps=3):
    """The bar a PyTorch user sees today: the oracle port (the reference's own torch ops) run eagerly on the SAME GPU
    through cuDNN, fp32 (TF32 as torch defaults: cudnn.allow_tf32=True) and fp16-autocast, cudnn.benchmark=True as
    test.py:148 sets it.  All 20 backbone calls + 12 ConvLSTM calls per window, CUDA-event timed."""
    from oracle import bin_oracle as O
    prev = torch.backends.cudnn.benchmark
    torch.backends.cudnn.benchmark = True
    sd = {k: v.to(dev) for k, v in O.synth_state_dict(0).items()}
    fr = [f.to(dev) for f in O.synth_frames(6, 1, H, W, seed=1234, smooth=True)]
    res = {}
    try:
        for tag, ctx in (("fp32", torch.autocast("cuda", enabled=False)),
                         ("fp16_autocast", torch.autocast("cuda", dtype=torch.float16))):
            with torch.no_grad(), ctx:
                for _ in range(2):
                    O.window_forward(fr, sd)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(steps):
                    O.window_forward(fr, sd)
                e1.record()
                torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / steps
            res[tag] = {"ms_per_window": ms, "windows_per_s": 1e3 / ms}
    finally:
        torch.backends.cudnn.benchmark = prev
    res["note"] = ("oracle port (same torch ops as the reference's RDN.py) eager on this GPU via cuDNN, cudnn.benchmark=True "
                   f"(test.py:148), tf32={bool(torch.backends.cudnn.allow_tf32)}; {steps} timed windows each")
    del sd, fr
    torch.cuda.empty_cache()
    return res


def run_reference_cuda(args):
    import torch
    dev = torch.device("cuda", 0)
    res = eager_cuda_numbers(torch, dev, args.height, args.width, steps=max(2, args.steps))
    print(json.dumps({"impl": "reference-port-eager-cuda", "metric": METRIC, "unit": UNIT,
                      "config": {"workload": f"bin_stage4 6-frame window {args.width}x{args.height}"}, **res}), flush=True)


# ------------------------------------------------------------------------------------------------
def _time_ms(torch, fn, reps=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def dominant_kernel_roofline(torch, ops, pk, ncalls, h, w):
    """The x-stacked RDB 3x3 convs 0..2 (conv_igemm_kernel<32,3,P8,SX>; the 4th conv runs inside the fused tail kernel)
    timed alone with CUDA events at the exact shapes the window launches them with (B = batched calls).  Also times the
    second-largest kernel, the fused RDB tail, against the HBM roofline, and the memory-bound K3/K4/K5 kernels."""
    dev = "cuda"
    tot_flops = tot_ms = 0.0
    x = torch.randn(ncalls, 12, h, w, 8, device=dev).half()
    g = torch.randn(ncalls, 16, h, w, 8, device=dev).half()
    for c in range(3):
        cin = 96 + 32 * c
        wt = torch.randn(32, cin, 3, 3, device=dev) / (cin * 9) ** 0.5
        wp, bp = ops.pack_conv_weight(wt, 32, cin), ops.pad_bias(torch.zeros(32, device=dev), 32)
        kw = dict(in0_planes=12, in1=g, in1_planes=4 * c, relu=True, out=g, out_plane0=4 * c)
        tot_ms += _time_ms(torch, lambda: ops.conv_fwd(x, wp, bp, 3, 32, **kw))
        tot_flops += 2.0 * ncalls * h * w * cin * 32 * 9
    ach = tot_flops / (tot_ms * 1e-3) / 1e12
    peak = pk["bf16_tflops"]
    # fused tail: conv3 (192 -> 32, 3x3, ReLU) + LFF (224 -> 96, 1x1) + residual; HBM sees x + g0..g2 in, x' out
    w3 = ops.pack_conv_weight(torch.randn(32, 192, 3, 3, device=dev) / 1728 ** 0.5, 32, 192)
    wl = ops.pack_conv_weight(torch.randn(96, 224, 1, 1, device=dev) / 224 ** 0.5, 96, 224)
    b3, bl = ops.pad_bias(torch.zeros(32, device=dev), 32), ops.pad_bias(torch.zeros(96, device=dev), 96)
    out = torch.empty(ncalls, 12, h, w, 8, device=dev).half()
    tail_ms = _time_ms(torch, lambda: ops.rdb_tail_fwd(x, g, w3, b3, wl, bl, out))
    tail_bytes = ncalls * h * w * (384 + 192)
    tail_flops = 2.0 * ncalls * h * w * (192 * 32 * 9 + 224 * 96)
    hbm = pk["hbm_gbs"]
    tail = {"bound": "hbm", "kernel": "rdb_tail (conv3 + LFF + residual fused)",
            "achieved": tail_bytes / (tail_ms * 1e-3) / 1e9, "peak": hbm, "unit": "GB/s",
            "frac": tail_bytes / (tail_ms * 1e-3) / 1e9 / hbm,
            "algorithmic_bytes_per_launch": tail_bytes,
            "tflops": tail_flops / (tail_ms * 1e-3) / 1e12, "tensor_frac": tail_flops / (tail_ms * 1e-3) / 1e12 / peak,
            "ms_per_launch": tail_ms}
    # memory-bound kernels of the path (north_star: K3 packer, K5 ConvLSTM), algorithmic bytes per SURVEY 8d
    H, W = 2 * h, 2 * w
    frames = [[torch.rand(1, 3, H, W, device=dev) for _ in range(2)] for _ in range(ncalls)]
    pack_ms = _time_ms(torch, lambda: ops.pack_frames(frames))
    pack_bytes = ncalls * H * W * (2 * 3 * 4) + ncalls * h * w * 32 * 2           # fp32 frames in, 32 fp16 channels out
    xl = torch.rand(1, 3, H, W, device=dev)
    wl_, bl_ = torch.randn(12, 6, 3, 3, device=dev) * 0.1, torch.zeros(12, device=dev)
    lstm_ms = _time_ms(torch, lambda: ops.convlstm_fwd(xl, wl_, bl_, None))
    lstm_bytes = H * W * 3 * 4 * 3                                                 # x in; h', c' out (prev_state = None)
    mem = {"pack_frames(K3)": {"ms": pack_ms, "GBps": pack_bytes / (pack_ms * 1e-3) / 1e9, "frac": pack_bytes / (pack_ms * 1e-3) / 1e9 / hbm,
                               "algorithmic_bytes": pack_bytes},
           "convlstm(K5, state=None)": {"ms": lstm_ms, "GBps": lstm_bytes / (lstm_ms * 1e-3) / 1e9,
                                        "frac": lstm_bytes / (lstm_ms * 1e-3) / 1e9 / hbm, "algorithmic_bytes": lstm_bytes}}
    return {"bound": "tensor", "kernel": "RDB 3x3 convs 0..2, x-stacked implicit GEMM (3 shapes)", "achieved": ach,
            "peak": peak, "unit": "TFLOP/s", "frac": ach / peak,
            # algorithmic: reads 5*230400*(192+256+320) B, writes 3*5*230400*64 B
            "algorithmic_bytes_per_launch_set": ncalls * h * w * (192 + 256 + 320) + 3 * ncalls * h * w * 64,
            "peak_source": f"bf16_tflops ({pk['source']}: H100 SXM data sheet unless MEASURED_PEAKS.json; kernel timed alone)",
            "algorithmic_flops_per_launch_set": tot_flops, "ms_per_launch_set": tot_ms,
            "second_kernel": tail,
            "memory_bound_kernels": mem}


def train_step_numbers(torch, dev, steps=4, warm=2, B=8, H=256, W=256, ddp=None):
    """BASELINE config 3: optimize_parameters (bin_model.py:130-141) on the shipped 6-frame net, batch 8 x 256x256:
    zero_grad, forward, get_loss (l1, 17 terms, fused), backward, Adam (one launch).  With `ddp` the module is wrapped
    in DistributedDataParallel (bin_model.py:39-41): the 45.8 MB gradient all-reduce runs bucketed under the backward."""
    from bin_b200 import rdn
    from bin_b200.loss import pixel_loss
    from bin_b200.optim import Adam
    from oracle import bin_oracle as O
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    net = net.to(dev).train()
    model = net
    if ddp:
        model = torch.nn.parallel.DistributedDataParallel(net, device_ids=[dev.index], bucket_cap_mb=50)
    opt = Adam(net.parameters(), lr=1e-4, betas=(0.9, 0.99))
    fr = [f.to(dev) for f in O.synth_frames(6, B, H, W, seed=1234, smooth=True)]
    gt = [f.to(dev) for f in O.synth_frames(14, B, H, W, seed=4321, smooth=True)]
    losses = []

    def step():
        opt.zero_grad(set_to_none=True)
        loss, _ = pixel_loss(model(*fr), gt, "l1")
        loss.backward()
        opt.step()
        return loss
    for _ in range(warm):
        losses.append(step().item())
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        l = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    losses.append(l.item())
    flops = 3 * 2.0 * MACS_PER_PX * B * H * W
    res = {"ms_per_step": ms, "config": f"optimize_parameters: 6-frame net, batch {B} x {W}x{H} per GPU, l1 (17 terms), Adam"
                                        + (", DistributedDataParallel (NCCL all-reduce of 45.8 MB overlapped with backward)" if ddp else ""),
           "tflops_3xF_fwd": flops / (ms * 1e-3) / 1e12, "losses": losses, "loss_decreases": losses[-1] < losses[0],
           "max_mem_GB": torch.cuda.max_memory_allocated(dev) / 2 ** 30}
    del net, model, opt, fr, gt
    torch.cuda.empty_cache()
    return res


DUMP_BYTES = 60 << 20                 # sample budget: with the .npy headers the files stay under 64 MB


def dump_outputs(out_dir, windows):
    """windows[i][k] = output k of window i of the last timed step -> out_dir/window<i>_out<k>.npy, float32.  When all
    outputs together exceed DUMP_BYTES, each one is reduced to the same fixed seeded sample of its flattened elements
    (sorted indices, generator seed 0), so two builds run with the same arguments write comparable files."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    n_all = sum(o.numel() for w_ in windows for o in w_)
    for i, w_ in enumerate(windows):
        for k, o in enumerate(w_):
            flat = o.detach().float().reshape(-1)
            cap = max(1, DUMP_BYTES // 4 // len(windows) // len(w_))
            if n_all * 4 > DUMP_BYTES and flat.numel() > cap:
                idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:cap].sort().values
                flat = flat[idx.to(flat.device)]
            np.save(os.path.join(out_dir, f"window{i}_out{k:02d}.npy"), flat.cpu().numpy().astype(np.float32))


def run_ours(args):
    import torch
    import torch.distributed as dist
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world != args.gpus:
        if world == 1 and args.gpus > 1:
            raise SystemExit("launch with torch.distributed.run --nproc-per-node N for --gpus N")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    nccl_init_ms = 0.0
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
        t0 = time.perf_counter()
        dist.all_reduce(torch.zeros(1, device=dev))                 # NCCL communicator set-up (lazy) -- NOT the broadcast
        torch.cuda.synchronize()
        nccl_init_ms = (time.perf_counter() - t0) * 1e3
    from bin_b200 import _lib, ops, rdn
    from bin_b200 import dist as bd
    from oracle import bin_oracle as O          # only for synthetic weights/inputs + cpu_baseline
    _lib.check(_lib.lib().bin_check_device())
    H, W, S = args.height, args.width, args.windows_per_step
    pk = peaks()

    torch.manual_seed(1000 + rank)              # ranks differ until the broadcast
    net = rdn.bin_stage4_lstm()
    if rank == 0:
        net.load_state_dict(O.synth_state_dict(0), strict=True)
    net = net.to(dev).eval()
    torch.cuda.synchronize()
    b0, b1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    b0.record()
    bcast_bytes = bd.broadcast_weights(net, src=0)          # the single collective (NCCL over NVLink)
    b1.record()
    torch.cuda.synchronize()
    bcast_ms = b0.elapsed_time(b1)

    # S independent windows per step, all resident (device) / pinned (host)
    wins_host = [[f.pin_memory() for f in O.synth_frames(6, 1, H, W, seed=1234 + 97 * rank + i, smooth=True)] for i in range(S)]
    wins_dev = [[f.to(dev) for f in w_] for w_ in wins_host]

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    sampler = ClockSampler(local)
    sampler.start()                              # NVML start-up happens here, long before the timed region
    with torch.no_grad():
        outs = None
        for _ in range(args.warmup):
            for w_ in wins_dev:
                outs = net(*w_)                  # same statement as the timed loop: the previous window's 14 outputs stay alive
                                                 # while the next window allocates its own, so the caching allocator reaches
                                                 # its steady state here (a one-off 220 ms of cudaMalloc fell into the FIRST
                                                 # timed step when the warm-up discarded its outputs: step_ms 365, 144, 144, ...)
        # Settle: a box that has been idle (the reference arm runs on the CPU first) starts at the maximum clock and the
        # power governor then swings below its steady state for a few seconds (seen as a first bench process 6-12 % slower
        # than every later one on the same box, with `e2e` -- measured later in the same process -- FASTER than the
        # device-resident value).  Keep running untimed steps for at least 2.5 s and until three consecutive steps agree within
        # 1.5 % (at most ~6 s); the timed region below is still exactly --steps steps, and what was run here is reported in the line.
        settle_ms = []
        t_settle = time.perf_counter()
        while time.perf_counter() - t_settle < 6.0:
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            for w_ in wins_dev:
                outs = net(*w_)
            s1.record()
            s1.synchronize()
            settle_ms.append(s0.elapsed_time(s1))
            last = settle_ms[-3:]
            if time.perf_counter() - t_settle >= 2.5 and max(last) - min(last) <= 0.015 * min(last):
                break
        barrier()
        sampler.mark_begin()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        marks = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps)]   # one per step boundary, never waited on in the loop
        e0.record()
        for i in range(args.steps):
            for w_ in wins_dev:
                outs = net(*w_)
            marks[i].record()
        e1.record()
        barrier()
        sampler.mark_end()
        ms_dev = e0.elapsed_time(e1)
        step_ms = [a.elapsed_time(b) for a, b in zip([e0] + marks[:-1], marks)]
        clocks = sampler.stop()
        if args.dump_outputs and rank == 0:
            # the last step's windows once more, untimed (keeping all their outputs alive inside the timed region would
            # add allocations to it); the path is deterministic, which the last window's timed outputs confirm bit for bit
            last_step = [net(*w_) for w_ in wins_dev]
            if not all(torch.equal(a, b) for a, b in zip(last_step[-1], outs)):
                raise SystemExit("--dump-outputs: re-running the last step did not reproduce its timed outputs")
            dump_outputs(args.dump_outputs, last_step)
            del last_step
        # ---- end-to-end: pinned host -> device, forward, 3 result images -> pinned host -----------
        from bin_b200.pipeline import WindowPipeline
        pipe = WindowPipeline(net, dev)
        out_sets = [[torch.empty((1, 3, H, W), dtype=torch.float32).pin_memory() for _ in range(3)] for _ in range(2)]
        for i in range(max(2, args.warmup // 2)):
            pipe.submit(wins_host[i % S], out_sets[i % 2])
        pipe.drain()
        barrier()
        e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e2.record()
        n = 0
        for _ in range(args.steps):
            for w_ in wins_host:
                pipe.submit(w_, out_sets[n % 2])
                n += 1
        pipe.drain()
        e3.record()
        barrier()
        ms_e2e = e2.elapsed_time(e3)
        e2e_ok = bool(torch.equal(out_sets[(n - 1) % 2][0], outs[13].cpu()))
    finite = bool(all(torch.isfinite(t).all() for t in outs))
    # per-rank record (the driver computes scaling from `value`; this shows WHICH rank bounds it)
    per_rank = [{"rank": rank, "gpu": local, "ms_per_step": ms_dev / args.steps, "e2e_ms_per_step": ms_e2e / args.steps,
                 "clocks": clocks,
                 "step_ms": {"min": round(min(step_ms), 2), "median": round(sorted(step_ms)[len(step_ms) // 2], 2),
                             "max": round(max(step_ms), 2), "first3": [round(x, 2) for x in step_ms[:3]],
                             "last3": [round(x, 2) for x in step_ms[-3:]]},
                 "settle": {"untimed_steps": len(settle_ms), "first_ms": round(settle_ms[0], 2), "last_ms": round(settle_ms[-1], 2),
                            "slowest_ms": round(max(settle_ms), 2)}}]
    if world > 1:
        gathered = [None] * world
        dist.all_gather_object(gathered, per_rank[0])
        per_rank = gathered
    ms_dev = max(r["ms_per_step"] for r in per_rank) * args.steps
    ms_e2e = max(r["e2e_ms_per_step"] for r in per_rank) * args.steps

    train_ddp = None
    if world > 1 and not args.no_extras:
        # training-side multi-GPU number (SURVEY 8e): one bucketed gradient all-reduce per step under DDP
        t = train_step_numbers(torch, dev, steps=3, warm=2, ddp=True)
        tm = [None] * world
        dist.all_gather_object(tm, t["ms_per_step"])
        train_ddp = dict(t, ms_per_step=max(tm), per_rank_ms=tm,
                         samples_per_s=world * 8 / (max(tm) * 1e-3))

    extras = {}
    if rank == 0 and world == 1 and not args.no_extras:
        from bin_b200.streaming import StreamingBIN, tensor2img_u8, test_py_padding, upload_frame_u8
        with torch.no_grad():
            pad = test_py_padding(H, W)
            gen = torch.Generator().manual_seed(7)
            nst = 12
            vid = [torch.randint(0, 256, (H, W, 3), generator=gen, dtype=torch.uint8).pin_memory() for _ in range(6 + 3 + nst)]
            st = StreamingBIN(net)
            host_out = [torch.empty((H, W, 3), dtype=torch.uint8).pin_memory() for _ in range(3)]
            nwin = 0
            for i, img in enumerate(vid):
                if i == 6 + 3:
                    torch.cuda.synchronize()
                    t_s = time.perf_counter()
                o = st.push(upload_frame_u8(img, pad, dev))
                if o is not None:
                    for dst, k in zip(host_out, (13, 8, 12)):
                        dst.copy_(tensor2img_u8(o[k], crop=(pad[2], pad[0], H, W)), non_blocking=True)
                    nwin += 1 if i >= 6 + 3 else 0
            torch.cuda.synchronize()
            dt = time.perf_counter() - t_s
            extras["streaming"] = {"value": nwin / dt, "unit": UNIT, "windows": nwin,
                                   "padded_hw": [H + pad[2] + pad[3], W + pad[0] + pad[1]],
                                   "note": "StreamingBIN on test.py-padded frames (768x1344 for 720p): uint8 HWC upload once per frame, "
                                           "stage-1 reuse (13 backbone calls per window), uint8 crops of outputs 13/8/12 downloaded"}
            del st, vid
            # fp32-accurate mode (north_star's 1e-5 bar): same kernels, split-fp16 x3
            rdn.set_precision(net, "fp32")
            for _ in range(2):
                net(*wins_dev[0])
            ms32 = _time_ms(torch, lambda: net(*wins_dev[0]), reps=4, warm=0)
            rdn.set_precision(net, "fp16")
            extras["fp32_mode"] = {"value": 1e3 / ms32, "unit": UNIT, "ms_per_window": ms32,
                                   "note": "set_precision(net, 'fp32'): split-fp16 x3 on the same wgmma kernels, <= 1e-5 vs the fp32 oracle (tests)"}
        rdn.release_workspaces()
        torch.cuda.empty_cache()
        extras["eager_cuda"] = eager_cuda_numbers(torch, dev, H, W)
        extras["train_step"] = train_step_numbers(torch, dev)
        # CPU baseline: bounded sample = ONE real quarter-area window (same aspect), scaled x4 by pixel count; the
        # `--impl reference` arm times full-size windows
        run, kind = cpu_window_runner()
        threads, sweep = pick_cpu_threads(run, budget_s=10.0)
        sh, sw = H // 2, W // 2
        crop = [f[:, :, :sh, :sw].contiguous() for f in wins_host[0]]
        t0 = time.perf_counter()
        run(crop)
        cpu_dt = time.perf_counter() - t0
        scale = (H * W) / float(sh * sw)
        extras["cpu_baseline"] = {"value": 1.0 / (cpu_dt * scale), "unit": UNIT, "cores": threads, "kind": kind,
                                  "host_cores": os.cpu_count(), "thread_sweep_192x320_s": sweep,
                                  "sample": f"one {sw}x{sh} 6-frame window ({cpu_dt:.1f} s of CPU), scaled x{scale:.0f} by pixel "
                                            f"count to {W}x{H}; `--impl reference` times full-size windows"}
    if rank == 0 and not args.no_extras:
        rdn.release_workspaces()
        torch.cuda.empty_cache()
        extras["roofline"] = dominant_kernel_roofline(torch, ops, pk, 5, H // 2, W // 2)
    if rank == 0:
        ms_step = ms_dev / args.steps
        value = world * S / (ms_step * 1e-3)
        e2e_val = world * S / (ms_e2e / args.steps * 1e-3)
        flops = 2.0 * MACS_PER_PX * H * W * S
        line = {
            "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms_step, "ms_per_window": ms_step / S, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f16", "data": "synthetic",
            "config": {"workload": f"bin_stage4 6-frame window {W}x{H} (SURVEY 8d config 2b; what test.py runs)",
                       "frames": 6, "windows_per_gpu_per_step": S, "outputs": 14,
                       "arithmetic": "fp16 operands / fp32 accumulate (wgmma f32.f16.f16), fp32 frames in/out, fp32 ConvLSTM",
                       "warmup_policy": "--warmup steps, then untimed settle steps (>= 2.5 s, until 3 consecutive steps agree within 1.5 %, <= 6 s; per_rank[].settle) so that the timed steps see the governor's steady state",
                       "l2": f"{S} distinct windows per step, per-window working set (>1 GB of activations per backbone stage) >> 50 MB L2; no explicit flush",
                       "executed_flop_fraction": EXECUTED_FRACTION, "weights": "synthetic U(+-1/sqrt(fan_in)) seed 0",
                       "nccl_init_ms": nccl_init_ms, "weight_broadcast_ms": bcast_ms, "weight_broadcast_bytes": bcast_bytes},
            "window_tflops_reference_as_executed": flops / (ms_step * 1e-3) / 1e12,
            "window_frac_of_peak_sustained": flops / (ms_step * 1e-3) / 1e12 / pk["bf16_tflops_sustained"],
            "frames_per_s": value * 14,
            "e2e": {"value": e2e_val, "unit": UNIT, "h2d_bytes_per_step": S * 6 * 3 * H * W * 4, "d2h_bytes_per_step": S * 3 * 3 * H * W * 4,
                    "note": "WindowPipeline: pinned-host frames in, outputs 13,8,12 (test.py:380-402) back to pinned host, copies overlapped with the previous/next window",
                    "matches_device_result": e2e_ok},
            "gpu_launches": args.steps * S * LAUNCHES_PER_WINDOW * 2,
            "gpu_launches_note": f"per window: 4 batched backbone stages x (1 pack + 42 conv + 12 fused RDB tails) + 3 ConvLSTM launches (6 cells) = {LAUNCHES_PER_WINDOW} kernels "
                                 "(replayed as one CUDA graph); timed twice (value, e2e)",
            "per_rank": per_rank,
            "clocks": per_rank[0]["clocks"], "outputs_finite": finite,
        }
        if train_ddp is not None:
            line["train_step_ddp"] = train_ddp
        line.update(extras)
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "reference-cuda"])
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--windows-per-step", type=int, default=5)
    ap.add_argument("--no-extras", action="store_true", help="skip roofline / cpu_baseline / eager / train extras")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the outputs of the last timed step to DIR/*.npy (float32, <= 64 MB in all; recomputed after the "
                         "timed region, so the timing is that of a run without the flag)")
    args = ap.parse_args()
    if args.impl == "reference-cuda":
        run_reference_cuda(args)
    elif args.impl == "reference":
        run_reference(args)
    else:
        args.warmup = max(args.warmup, 3)
        run_ours(args)


if __name__ == "__main__":
    main()
