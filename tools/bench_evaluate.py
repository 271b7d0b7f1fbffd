"""Windows per second of test.py's test-set evaluation: (a) a restatement of test.py's serial loop (one module call per
window, tensor2img on the host, cv2.imwrite through png.install_cv2_imwrite, cv2 re-reads, the bin_b200.metrics
drop-ins), (b) evaluate.evaluate_testset on one GPU, (c) evaluate_testset on every visible GPU (one process each, NCCL).

The test set is a seeded 1280x720 PNG tree built in a temporary directory (default 2 folders x 21 blurry frames = 40
windows, GT frames at the 240 fps names), the weights are synthetic.  (a) and (b) alternate after one warm-up run of
each; each run writes into a fresh output directory.  The GPU-busy fraction of (b) is the CUDA-event time of the same
windows' device work (stream_video, crops, batched metrics, PNG encodes) with every frame already on the device, over
(b)'s wall time.  Prints one JSON line (and writes it to --json when given).

    python tools/bench_evaluate.py [--folders 2] [--frames 21] [--repeats 2] [--json out.json]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import bin_oracle as O  # noqa: E402

H, W, FIRST = 720, 1280, 17


def make_tree(root, folders, frames, seed=5):
    import cv2
    g = np.random.default_rng(seed)
    for k in range(folders):
        folder = f"clip{k:02d}"
        for sub in ("in", "gt"):
            os.makedirs(os.path.join(root, sub, folder))
        base = g.integers(0, 256, size=(H // 8, W // 8, 3)).astype(np.float32)
        for num in range(FIRST, FIRST + 8 * (frames - 1) + 13):
            base += g.normal(0, 2, size=base.shape).astype(np.float32)
            gt = np.clip(cv2.resize(base, (W, H), interpolation=cv2.INTER_CUBIC), 0, 255).astype(np.uint8)
            cv2.imwrite(os.path.join(root, "gt", folder, f"{num:05d}.png"), gt)
            if (num - FIRST) % 8 == 0 and (num - FIRST) // 8 < frames:
                cv2.imwrite(os.path.join(root, "in", folder, f"{num:05d}.png"), cv2.GaussianBlur(gt, (9, 9), 3.0))
    return os.path.join(root, "in"), os.path.join(root, "gt")


def make_net(device="cuda"):
    from bin_b200 import rdn
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    return net.to(device).eval()


def test_py_loop(net, inp, gt, out):
    """test.py:222-458 restated with the GPU drop-ins: -> windows run."""
    import cv2
    from bin_b200 import metrics as M
    from bin_b200.png import install_cv2_imwrite
    from bin_b200.streaming import test_py_padding
    install_cv2_imwrite()
    rd = lambda p: cv2.imread(p)[:, :, [2, 1, 0]]                                  # noqa: E731
    tensor2img = lambda t: O.tensor2img_bgr_u8(t.squeeze(0))                       # noqa: E731 (util.tensor2img: host)
    nwin = 0
    for dir in sorted(os.listdir(inp)):
        os.makedirs(os.path.join(out, dir))
        frames = sorted(os.listdir(os.path.join(inp, dir)))
        first = int(frames[0][:-4])
        L = len(frames) - 1
        for index, frame in enumerate(frames[:-1]):
            pos = [max(index - 2, 0), max(index - 1, 0), min(index, L), min(index + 1, L), min(index + 2, L), min(index + 3, L)]
            paths = [os.path.join(inp, dir, f"{first + 8 * p:05d}.png") for p in pos]
            imgs = [cv2.imread(p) for p in paths]
            h, w = imgs[0].shape[:2]
            pl, pr, pt, pb = test_py_padding(h, w)
            pad = torch.nn.ReplicationPad2d([pl, pr, pt, pb])
            data = [pad(O.read_image_u8(im).cuda().unsqueeze(0)) for im in imgs]
            with torch.no_grad():
                Ft_p = net(*data)
            crop = lambda t: tensor2img(t)[pt:pt + h, pl:pl + w, :]                # noqa: E731
            y_, x0_s, x1_s, s2, s3 = (crop(Ft_p[k]) for k in (13, 8, 12, 7, 9))
            num = int(frame[:-4])
            o_mid, o_first, o_second = (os.path.join(out, dir, f"{num + d:05d}.png") for d in (8, 4, 12))
            g_mid, g_first, g_second = (os.path.join(gt, dir, f"{num + d:05d}.png") for d in (8, 4, 12))
            cv2.imwrite(o_mid, y_)
            if index < L - 1 and not os.path.exists(o_second):
                cv2.imwrite(o_second, x1_s)
                res, g_ = rd(o_second), rd(g_second)
                M.compare_psnr(res, g_), M.compare_ssim(res, g_, multichannel=True)
            if not os.path.exists(o_first):
                cv2.imwrite(o_first, x0_s)
                res, g_ = rd(o_first), rd(g_first)
                M.compare_psnr(res, g_), M.compare_ssim(res, g_, multichannel=True)
            rec, g_ = rd(o_mid), rd(g_mid)
            diff = 128.0 + rec - g_
            np.mean(np.abs(diff - 128.0)), math.log10(255.0 / math.sqrt(np.mean((diff - 128.0) ** 2)))
            M.compare_psnr(rec, g_), M.compare_ssim(rec, g_, multichannel=True)
            blur = rd(paths[3])
            M.compare_psnr(blur, g_), M.compare_ssim(blur, g_, multichannel=True)
            nwin += 1
    return nwin


def device_seconds(net, inp, gt):
    """CUDA-event time of the evaluator's device work with every frame resident: the GPU-busy numerator."""
    import cv2
    from bin_b200 import rdn
    from bin_b200.evaluate import _scored
    from bin_b200.metrics import image_metrics_batch
    from bin_b200.png import encode_png_async
    from bin_b200.streaming import stream_video, tensor2img_u8, test_py_padding, test_py_writes, upload_frame_u8
    rdn.set_outputs(net, (13, 8, 12))
    total = 0.0
    try:
        for dir in sorted(os.listdir(inp)):
            names = sorted(os.listdir(os.path.join(inp, dir)))
            n, first = len(names), int(names[0][:-4])
            u8 = [torch.from_numpy(cv2.imread(os.path.join(inp, dir, x))).cuda() for x in names]
            gts = {k: torch.from_numpy(cv2.imread(os.path.join(gt, dir, f"{first + 8 * (k // 3) + 4 * (k % 3 + 1):05d}.png"))).cuda()
                   for k in range(3 * (n - 1))}
            h, w = u8[0].shape[:2]
            pad = test_py_padding(h, w)
            frames = [upload_frame_u8(x, pad, "cuda") for x in u8]
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            pend = []
            for i, outs in stream_video(net, iter(frames)):
                todo = test_py_writes(i, n)
                imgs = {k: tensor2img_u8(outs[k], crop=(pad[2], pad[0], h, w)) for k in todo}
                g = {13: gts[3 * i + 1], 8: gts[3 * i], 12: gts[3 * i + 2]}
                pairs = [(imgs[k], g[k]) if k >= 0 else (u8[min(i + 1, n - 1)], g[13]) for k in _scored(i, n)]
                pend.append((image_metrics_batch(pairs, bgr=True), encode_png_async([imgs[k] for k in todo])))
            t1.record()
            torch.cuda.synchronize()
            total += t0.elapsed_time(t1) / 1e3
    finally:
        rdn.set_outputs(net, None)
    return total


def _world_worker(rank, world, inp, gt, out, port):
    import torch.distributed as tdist
    from bin_b200 import dist as bdist
    from bin_b200.evaluate import evaluate_testset
    torch.cuda.set_device(rank)
    tdist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        net = make_net(f"cuda:{rank}")
        bdist.broadcast_weights(net)
        evaluate_testset(net, inp, gt, out, "bin")
    finally:
        tdist.destroy_process_group()


def all_gpus(inp, gt, out, world):
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    t = time.perf_counter()
    mp.spawn(_world_worker, args=(world, inp, gt, out, port), nprocs=world, join=True)
    return time.perf_counter() - t


def log(msg):
    print(f"bench_evaluate: {msg}", file=sys.stderr, flush=True)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError) as e:
        return [f"nvidia-smi unavailable: {e}"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--folders", type=int, default=2)
    ap.add_argument("--frames", type=int, default=21)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_evaluate: no CUDA device (there is no CPU path to time)")
    from bin_b200.evaluate import evaluate_testset
    res = {"host_cores": os.cpu_count(), "host_cores_usable": len(os.sched_getaffinity(0)),
           "gpus_visible": torch.cuda.device_count(), "gpu_before": gpu_info()}
    with tempfile.TemporaryDirectory() as tmp:
        t = time.perf_counter()
        inp, gt = make_tree(os.path.join(tmp, "data"), args.folders, args.frames)
        res["tree_seconds"] = round(time.perf_counter() - t, 1)
        log(f"tree built in {res['tree_seconds']} s")
        nwin = args.folders * (args.frames - 1)
        net = make_net()
        runs = {"a": [], "b": []}
        k = 0

        def run(kind):
            nonlocal k
            k += 1
            out = os.path.join(tmp, f"out{k}")
            torch.cuda.synchronize()
            t = time.perf_counter()
            if kind == "a":
                assert test_py_loop(net, inp, gt, out) == nwin
            else:
                evaluate_testset(net, inp, gt, out, "bin")
            torch.cuda.synchronize()
            rate = nwin / (time.perf_counter() - t)
            log(f"run {k} ({kind}): {rate:.3f} windows/s")
            return rate

        run("a"), run("b")                                          # warm-up
        for _ in range(args.repeats):
            for kind in ("a", "b"):
                runs[kind].append(run(kind))
        dev_s = [device_seconds(net, inp, gt) for _ in range(2)][-1]
        world = torch.cuda.device_count()
        c = [nwin / all_gpus(inp, gt, os.path.join(tmp, f"c{r}"), world) for r in range(2)] if world > 1 else None
    med = {kk: statistics.median(v) for kk, v in runs.items()}
    res.update({
        "windows": nwin, "frame": f"{W}x{H}",
        "a_test_py_loop_windows_per_s": {"median": round(med["a"], 3), "runs": [round(x, 3) for x in runs["a"]]},
        "b_evaluator_1gpu_windows_per_s": {"median": round(med["b"], 3), "runs": [round(x, 3) for x in runs["b"]]},
        "b_over_a": round(med["b"] / med["a"], 2),
        "b_gpu_busy_fraction": round(dev_s * med["b"] / nwin, 3),
        "b_device_seconds": round(dev_s, 3),
        "c_evaluator_all_gpus_windows_per_s": ([round(x, 3) for x in c] if c else
                                               "same as (b): one GPU visible"),
        "gpu_after": gpu_info(),
    })
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
