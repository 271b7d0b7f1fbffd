"""Images written per second by demo.py's conversion: (a) a restatement of demo.py's serial loop (one module call per
window and per j, six cv2.imread and a replicate-pad per window, tensor2img on the host, png.imwrite), (b) demo.run_demo
on one GPU, (c) run_demo on every visible GPU (one process each, NCCL).

The input is a seeded 1280x720 folder of blurry frames built in a temporary directory (default 1 folder x 21 frames =
20 windows), the weights are synthetic, time_step is 0.5 unless --time_step says otherwise.  (a) and (b) alternate after
one warm-up run of each; each run writes into a fresh output directory.  Prints one JSON line (and writes it to --json
when given).

    python tools/bench_demo.py [--folders 1] [--frames 21] [--time_step 0.5] [--repeats 3] [--json out.json]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import bin_oracle as O  # noqa: E402
from tools.bench_evaluate import gpu_info, make_net  # noqa: E402

H, W, FIRST = 720, 1280, 17


def make_folder(root, folders, frames, seed=5):
    import cv2
    g = np.random.default_rng(seed)
    for k in range(folders):
        folder = os.path.join(root, f"clip{k:02d}")
        os.makedirs(folder)
        base = g.integers(0, 256, size=(H // 8, W // 8, 3)).astype(np.float32)
        for p in range(frames):
            base += g.normal(0, 2, size=base.shape).astype(np.float32)
            img = np.clip(cv2.resize(base, (W, H), interpolation=cv2.INTER_CUBIC), 0, 255).astype(np.uint8)
            cv2.imwrite(os.path.join(folder, f"{FIRST + 8 * p:05d}.png"), cv2.GaussianBlur(img, (9, 9), 3.0))
    return root


def demo_py_loop(net, inp, out, time_step):
    """demo.py:164-324 restated with the one-image GPU PNG drop-in: -> files written."""
    import cv2
    from bin_b200.demo import demo_py_steps
    from bin_b200.png import imwrite
    from bin_b200.streaming import test_py_padding
    tensor2img = lambda t: O.tensor2img_bgr_u8(t.squeeze(0))                       # noqa: E731 (util.tensor2img: host)
    steps = demo_py_steps(time_step)
    files = 0
    for dir in sorted(os.listdir(inp)):
        os.makedirs(os.path.join(out, dir))
        frames = sorted(os.listdir(os.path.join(inp, dir)))
        first = int(frames[0][:-4])
        L = len(frames) - 1
        for index, frame in enumerate(frames[:-1]):
            pos = [max(index - 2, 0), max(index - 1, 0), min(index, L), min(index + 1, L), min(index + 2, L), min(index + 3, L)]
            num = int(frame[:-4])
            o_first, o_second = (os.path.join(out, dir, f"{num + d:05d}.png") for d in (4, 12))
            for j in steps:
                imgs = [cv2.imread(os.path.join(inp, dir, f"{first + 8 * p:05d}.png")) for p in pos]
                h, w = imgs[0].shape[:2]
                pl, pr, pt, pb = test_py_padding(h, w)
                pad = torch.nn.ReplicationPad2d([pl, pr, pt, pb])
                data = [pad(O.read_image_u8(im).cuda().unsqueeze(0)) for im in imgs]
                o_mid = os.path.join(out, dir, f"{num + 5 + j:05d}.png")
                with torch.no_grad():
                    Ft_p = net(*data)
                crop = lambda t: tensor2img(t)[pt:pt + h, pl:pl + w, :]            # noqa: E731
                y_, x0_s, x1_s = (crop(Ft_p[k]) for k in (13, 8, 12))
                imwrite(o_mid, y_)
                files += 1
                if index < L - 1 and not os.path.exists(o_second):
                    imwrite(o_second, x1_s)
                    files += 1
                if not os.path.exists(o_first):
                    imwrite(o_first, x0_s)
                    files += 1
    return files


def _world_worker(rank, world, inp, out, time_step, port):
    import torch.distributed as tdist
    from bin_b200 import dist as bdist
    from bin_b200.demo import run_demo
    torch.cuda.set_device(rank)
    tdist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        net = make_net(f"cuda:{rank}")
        bdist.broadcast_weights(net)
        run_demo(net, inp, out, time_step=time_step, verbose=False)
    finally:
        tdist.destroy_process_group()


def all_gpus(inp, out, time_step, world):
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    t = time.perf_counter()
    mp.spawn(_world_worker, args=(world, inp, out, time_step, port), nprocs=world, join=True)
    return time.perf_counter() - t


def log(msg):
    print(f"bench_demo: {msg}", file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--folders", type=int, default=1)
    ap.add_argument("--frames", type=int, default=21)
    ap.add_argument("--time_step", type=float, default=0.5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_demo: no CUDA device (there is no CPU path to time)")
    from bin_b200.demo import demo_py_writes, run_demo
    res = {"host_cores": os.cpu_count(), "host_cores_usable": len(os.sched_getaffinity(0)),
           "gpus_visible": torch.cuda.device_count(), "gpu_before": gpu_info(), "time_step": args.time_step}
    nwin = args.folders * (args.frames - 1)
    nfiles = args.folders * sum(len(v) for i in range(args.frames - 1)
                                for v in demo_py_writes(i, args.frames, args.time_step).values())
    with tempfile.TemporaryDirectory() as tmp:
        inp = make_folder(os.path.join(tmp, "in"), args.folders, args.frames)
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
                assert demo_py_loop(net, inp, out, args.time_step) == nfiles
            else:
                assert run_demo(net, inp, out, time_step=args.time_step, verbose=False).files == nfiles
            torch.cuda.synchronize()
            rate = nfiles / (time.perf_counter() - t)
            log(f"run {k} ({kind}): {rate:.3f} images/s")
            return rate

        run("a"), run("b")                                          # warm-up
        for _ in range(args.repeats):
            for kind in ("a", "b"):
                runs[kind].append(run(kind))
        world = torch.cuda.device_count()
        c = ([nfiles / all_gpus(inp, os.path.join(tmp, f"c{r}"), args.time_step, world) for r in range(2)]
             if world > 1 else None)
    med = {kk: statistics.median(v) for kk, v in runs.items()}
    res.update({
        "windows": nwin, "images": nfiles, "frame": f"{W}x{H}",
        "a_demo_py_loop_images_per_s": {"median": round(med["a"], 3), "runs": [round(x, 3) for x in runs["a"]]},
        "b_run_demo_1gpu_images_per_s": {"median": round(med["b"], 3), "runs": [round(x, 3) for x in runs["b"]]},
        "b_over_a": round(med["b"] / med["a"], 2),
        "c_run_demo_all_gpus_images_per_s": ([round(x, 3) for x in c] if c else "same as (b): one GPU visible"),
        "gpu_after": gpu_info(),
    })
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
