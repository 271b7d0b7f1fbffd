"""Sharp frames per second turned into the blurred dataset tree: (a) a restatement of
create_dataset_blur_N_frames_average.py's serial loop (per window, cv2.imread of each of its frames, a float32 NumPy
average truncated to uint8, cv2.imwrite; then the sharp copy and the list), (b) dataprep.build_dataset on one GPU.

The input is a seeded 352x640 tree of smooth moving frames built in a temporary directory (default 2 videos x 200
frames) and linked in as each run's full_sharp, so no run extracts; window_size is 11, as the Adobe240 recipe.  (a)
and (b) alternate after one warm-up run of each; each run writes a fresh tree.  The GPU-busy fraction is the device
time of (b)'s work alone (the same chunks' upload, average and encode from frames already in pinned memory, between
CUDA events) over (b)'s wall time.  Prints one JSON line (and writes it to --json when given).

    python tools/bench_dataprep.py [--videos 2] [--frames 200] [--repeats 3] [--json out.json]
"""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_evaluate import gpu_info  # noqa: E402

H, W, WS = 352, 640, 11


def log(msg):
    print(f"bench_dataprep: {msg}", file=sys.stderr, flush=True)


def make_frames(root, videos, frames, seed=4):
    import cv2
    from bin_b200.dataprep import frame_name
    g = np.random.default_rng(seed)
    stems = []
    for v in range(videos):
        stem = f"clip{v:02d}"
        os.makedirs(os.path.join(root, stem))
        base = g.integers(0, 256, size=(H // 8, W // 8, 3)).astype(np.float32)
        for k in range(frames):
            base += g.normal(0, 2, size=base.shape).astype(np.float32)
            img = np.clip(cv2.resize(base, (W, H), interpolation=cv2.INTER_CUBIC), 0, 255).astype(np.uint8)
            assert cv2.imwrite(os.path.join(root, stem, frame_name(k)), cv2.GaussianBlur(img, (5, 5), 1.5))
        stems.append(stem)
    return stems


def script_loop(root, stems, ws):
    """create_clips_overlap (:87-148) for each video, serially, as the script computes it."""
    import cv2
    from bin_b200.dataprep import frame_name, window_count
    r = int((ws - 1) / 2)
    for stem in stems:
        src = os.path.join(root, "full_sharp", stem)
        n = len(os.listdir(src))
        names = []
        for w in range(window_count(n)):
            mid = 16 + 8 * w
            acc = 0.0
            for loc in range(mid - r, mid + r + 1):
                acc = acc + cv2.imread(os.path.join(src, frame_name(loc))).astype("float32")
            os.makedirs(os.path.join(root, "test_blur", stem), exist_ok=True)
            assert cv2.imwrite(os.path.join(root, "test_blur", stem, frame_name(mid)), (acc / float(2 * r + 1)).astype("uint8"))
            names.append(frame_name(mid))
        shutil.copytree(src, os.path.join(root, "test", stem))
        os.makedirs(os.path.join(root, "test_list"), exist_ok=True)
        with open(os.path.join(root, "test_list", stem + "_im_list.txt"), "w") as fh:
            fh.write("\n".join(names))


def device_seconds(frames_root, stems, ws):
    """CUDA-event time of build_dataset's device work alone: per chunk, the upload of its frames from pinned memory,
    the average and the PNG encode (with its copy back), for every video."""
    import cv2
    from bin_b200 import dataprep as D
    from bin_b200.png import encode_png_async
    total = 0.0
    for stem in stems:
        src = os.path.join(frames_root, stem)
        n = len(os.listdir(src))
        host = torch.from_numpy(np.stack([cv2.imread(os.path.join(src, D.frame_name(k))) for k in range(n)])).pin_memory()
        mids = D.window_mids(n, ws)
        for rep in range(2):                                        # the first pass warms the encoder's shapes
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            pending = []
            for chunk, lo, hi in D.chunks(mids, ws, D.CHUNK_WINDOWS):
                dev = host[lo:hi + 1].to("cuda", non_blocking=True)
                out = D.blur_average(dev, ws, first_mid=chunk[0] - lo, nwin=len(chunk))
                pending.append(encode_png_async(list(out.unbind(0))))
            t1.record()
            for p in pending:
                p.result()
            torch.cuda.synchronize()
        total += t0.elapsed_time(t1) / 1e3
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=2)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--decode_threads", type=int, default=8)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dataprep: no CUDA device (there is no CPU path to time)")
    from bin_b200.dataprep import build_dataset
    res = {"host_cores": os.cpu_count(), "host_cores_usable": len(os.sched_getaffinity(0)), "gpu_before": gpu_info(),
           "videos": args.videos, "frames_per_video": args.frames, "frame": f"{W}x{H}", "window_size": WS,
           "decode_threads": args.decode_threads}
    nframes = args.videos * args.frames
    with tempfile.TemporaryDirectory() as tmp:
        frames_root = os.path.join(tmp, "frames")
        stems = make_frames(frames_root, args.videos, args.frames)
        lst = os.path.join(tmp, "list.txt")
        with open(lst, "w") as fh:
            fh.write("\n".join(s + ".mp4" for s in stems))
        runs = {"a": [], "b": []}
        k = 0

        def run(kind):
            nonlocal k
            k += 1
            root = os.path.join(tmp, f"run{k}")
            os.makedirs(root)
            os.symlink(frames_root, os.path.join(root, "full_sharp"))
            torch.cuda.synchronize()
            t = time.perf_counter()
            if kind == "a":
                script_loop(root, stems, WS)
            else:
                build_dataset(root, test_list=lst, window_size=WS, decode_threads=args.decode_threads)
            torch.cuda.synchronize()
            sec = time.perf_counter() - t
            shutil.rmtree(root)
            log(f"run {k} ({kind}): {nframes / sec:.1f} frames/s")
            return sec

        run("a"), run("b")                                          # warm-up
        for _ in range(args.repeats):
            for kind in ("a", "b"):
                runs[kind].append(run(kind))
        dev = device_seconds(frames_root, stems, WS)
    med = {kk: statistics.median(v) for kk, v in runs.items()}
    res.update({
        "a_script_loop_frames_per_s": {"median": round(nframes / med["a"], 1),
                                       "runs": [round(nframes / x, 1) for x in runs["a"]]},
        "b_build_dataset_frames_per_s": {"median": round(nframes / med["b"], 1),
                                         "runs": [round(nframes / x, 1) for x in runs["b"]]},
        "b_over_a": round(med["a"] / med["b"], 2),
        "b_device_seconds": round(dev, 4), "b_wall_seconds": round(med["b"], 4),
        "b_gpu_busy_fraction": round(dev / med["b"], 4),
        "gpu_after": gpu_info(),
    })
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
