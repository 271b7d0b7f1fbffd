"""Time the GPU PNG encoder (bin_b200.png) and the host work it saves, and print the card, its power limit and the
host's core count with the results (one JSON line per case).

    python tools/bench_png.py [--iters 200] [--warmup 20] [--windows 12]

Cases:
  kernel      bin_png_encode_u8 for n = 3 natural-like 720x1280 frames, back to back on device-resident images,
              CUDA events over --iters launches after --warmup; bytes moved = payload read + files written;
  imwrite     wall time per image of bin_b200.png.imwrite from numpy against cv2.imwrite (skipped without cv2),
              and the file sizes against cv2's;
  loop        host CPU seconds per window (time.process_time) of a StreamingBIN loop at 768x1344 that writes three
              images per window as test.py does: tensor2img_u8 + encode_png_async (files of window k written while
              window k+1 runs), against tensor2img on the host + cv2.imwrite (skipped without cv2).
Needs a CUDA device; there is no CPU fallback."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bin_b200 import _lib, png, rdn             # noqa: E402
from bin_b200.streaming import StreamingBIN, tensor2img_u8, test_py_padding, upload_frame_u8   # noqa: E402
from oracle import bin_oracle as O              # noqa: E402
from oracle import png_oracle as P              # noqa: E402
from test_gpu_png import make_image             # noqa: E402

H100_HBM_TBPS = 3.35


def card():
    q = "name,power.limit"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().split(",")]
    except Exception as e:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(), f"unknown ({e})"
    return {"name": name, "power_limit": power, "host_cores": os.cpu_count()}


def bench_kernel(iters, warm):
    L = _lib.lib()
    h, w, n = 720, 1280, 3
    imgs = [torch.from_numpy(make_image("natural", h, w, seed=20 + i)).cuda() for i in range(n)]
    stride = (int(L.bin_png_max_bytes(h, w)) + 255) // 256 * 256
    out = torch.empty(n * stride, dtype=torch.uint8, device="cuda")
    sizes = torch.empty(n, dtype=torch.int64, device="cuda")
    ws = torch.empty(int(L.bin_png_workspace_bytes(n, h, w)), dtype=torch.uint8, device="cuda")
    ptrs = (C.c_void_p * n)(*[x.data_ptr() for x in imgs])
    s = torch.cuda.current_stream().cuda_stream

    def run():
        _lib.check(L.bin_png_encode_u8(ptrs, n, h, w, out.data_ptr(), stride, sizes.data_ptr(), ws.data_ptr(),
                                       ws.numel(), s))
    for _ in range(warm):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    written = int(sizes.sum().item())
    moved = n * h * (3 * w + 1) + written
    return {"case": "kernel", "n": n, "shape": [h, w], "ms": round(ms, 4), "bytes_moved": moved,
            "hbm_share": round(moved / (ms * 1e-3) / (H100_HBM_TBPS * 1e12), 4), "file_bytes": sizes.tolist()}


def bench_imwrite(reps):
    try:
        import cv2
    except ImportError:
        cv2 = None
    rows = []
    d = tempfile.mkdtemp()
    for kind in ("natural", "noise"):
        img = make_image(kind, 720, 1280, seed=5)
        png.imwrite(os.path.join(d, "w.png"), img)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            png.imwrite(os.path.join(d, "g.png"), img)
        t_gpu = (time.perf_counter() - t0) / reps
        row = {"case": "imwrite", "kind": kind, "gpu_ms": round(t_gpu * 1e3, 2),
               "gpu_bytes": os.path.getsize(os.path.join(d, "g.png")), "cv2_like_bytes": P.cv2_like_size(img)}
        if cv2 is not None:
            t0 = time.perf_counter()
            for _ in range(reps):
                cv2.imwrite(os.path.join(d, "c.png"), img)
            row["cv2_ms"] = round((time.perf_counter() - t0) / reps * 1e3, 2)
            row["cv2_bytes"] = os.path.getsize(os.path.join(d, "c.png"))
        rows.append(row)
    return rows


def bench_loop(windows, mode):
    h, w = 768, 1344
    pl, pr, pt, pb = test_py_padding(h, w)
    net = rdn.bin_stage4_lstm()
    net.load_state_dict(O.synth_state_dict(0), strict=True)
    net = net.cuda().eval()
    frames = [torch.from_numpy(make_image("natural", h, w, seed=40 + i)).cuda() for i in range(windows + 5)]
    d = tempfile.mkdtemp()
    if mode == "cv2":
        import cv2
    st = StreamingBIN(net)
    pending = None
    cpu = []
    with torch.no_grad():
        for k, f in enumerate(frames):
            t0 = time.process_time()
            outs = st.push(upload_frame_u8(f, (pl, pr, pt, pb), "cuda"))
            if outs is not None:
                if mode == "gpu":
                    imgs = [tensor2img_u8(outs[j], crop=(pt, pl, h, w)) for j in (0, 1, 2)]
                    handle = png.encode_png_async(imgs)
                    if pending is not None:
                        for j, data in enumerate(pending.result()):
                            with open(os.path.join(d, f"{k}_{j}.png"), "wb") as fh:
                                fh.write(data)
                    pending = handle
                else:
                    for j in (0, 1, 2):
                        img = O.tensor2img_bgr_u8(outs[j][0].cpu())[pt:pt + h, pl:pl + w, :]
                        cv2.imwrite(os.path.join(d, f"{k}_{j}.png"), img)
                torch.cuda.synchronize()
                if k >= 7:                                  # after two warm-up windows
                    cpu.append(time.process_time() - t0)
    return {"case": "loop", "mode": mode, "shape": [h, w], "windows": len(cpu),
            "cpu_s_per_window": round(float(np.mean(cpu)), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--windows", type=int, default=12)
    a = ap.parse_args()
    print(json.dumps({"card": card()}))
    print(json.dumps(bench_kernel(a.iters, a.warmup)))
    for row in bench_imwrite(10):
        print(json.dumps(row))
    print(json.dumps(bench_loop(a.windows, "gpu")))
    try:
        import cv2  # noqa: F401
        print(json.dumps(bench_loop(a.windows, "cv2")))
    except ImportError:
        print(json.dumps({"case": "loop", "mode": "cv2", "skipped": "cv2 not importable"}))


if __name__ == "__main__":
    main()
