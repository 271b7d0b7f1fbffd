"""test.py's test-set evaluation (test.py:73-506) on one or more GPUs: the paper's Adobe240 table in one call.

evaluate_testset runs the windows test.py runs, in its order, over every folder of a test set, writes the three images
test.py writes per window and the two logs it writes, and computes every metric it logs:

  * windows are streamed per video (streaming.stream_video), each frame decoded once, on host threads that read ahead;
  * Ft_p[13], Ft_p[8] and Ft_p[12] (rdn.set_outputs) are cropped on the device (tensor2img_u8) and encoded by the GPU
    PNG encoder (png.encode_png_async); a host thread writes the files;
  * each window's scores are one batched metrics launch (metrics.image_metrics_batch) whose sums are read one window
    late, so the host never waits on the GPU between windows;
  * with several ranks, each runs a contiguous run of windows (dist.shard_test_set) and rank 0 writes the logs from
    the gathered records, in test.py's window order, so the logs do not depend on the number of ranks.

The scores are test.py's: it re-reads each PNG it writes, and the files decode to the pixels they were encoded from,
so scoring the device image is scoring the file.  test.py scores RGB arrays (read_image_np) and cv2 and tensor2img_u8
hold BGR; the SSIM sums run over the channels in order, so the metrics run with their BGR flag and give the bits of the
RGB view.  Where this departs from test.py:

  * the output directory must not hold any image it would write: test.py skips an existing file and then logs other
    metrics (test.py:376, 405, 418), so a partly written directory raises instead of being resumed;
  * test.py's `mse == 0: return 100.0` (test.py:440-441) ends main() without a summary: the logs stop at the same
    message and BinB200Error names the frame (the other windows' images are written all the same);
  * test.py's 1280x720 limit (test.py:345-346) is not imposed;
  * only time_step 0.5, the middle frame, exists (test.py:303-305 for this net);
  * the blurry frames of a folder must be named first, first + 8, ... (the Adobe240 test sets are): test.py names its
    inputs that way (test.py:262-287) but takes the GT names from the listing, and only such folders give one answer.

python -m bin_b200.evaluate takes test.py's arguments (see main()); under torchrun it shards over the ranks."""
from __future__ import annotations

import argparse
import collections
import concurrent.futures as cf
import logging
import math
import os
import time
from datetime import datetime
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch

from . import dist as bdist
from . import rdn
from ._lib import BinB200Error
from .metrics import image_metrics_batch
from .png import encode_png_async
from .streaming import (VideoPlan, stream_video, tensor2img_u8, test_py_names, test_py_padding, test_py_window,
                        test_py_writes, upload_frame_u8)

WANTED = (13, 8, 12)                    # the three outputs test.py writes (test.py:380-382)
RESULT_DIR = "60fps_test_results"       # test.py:112-119: round(1 / 0.5) * 30 fps
PAD = 32                                # test.py:128, logged as the padding mode
SSIM_MSG = "skimage.measure.ssim"       # test.py:31-37, use_default_ssim = 1


# ----------------------------------------------------------------------------- names (test.py:242-330)
class WindowPaths(NamedTuple):
    inputs: Tuple[str, ...]             # the six frames the window reads (test.py:334)
    gt: Dict[int, str]                  # output index -> its GT (test.py:324-326)
    out: Dict[int, str]                 # output index -> the file test.py writes it to (test.py:320, 329-330)
    blurry: str                         # the blurry frame scored against the middle GT (test.py:300, 452)


def window_paths(input_path: str, gt_path: str, gen_dir: str, folder: str, first: int, i: int, n: int,
                 direct_interp: bool = False) -> WindowPaths:
    """The paths window i of an n-frame folder whose first blurry frame is named `first` reads and writes in test.py:
    inputs named first + 8 * position (test.py:260-282), from gt_path with direct_interp; GT and output names from the
    window's blurry frame first + 8 i (test.py:287-299, 318-330)."""
    src = os.path.join(gt_path if direct_interp else input_path, folder)
    name = lambda num: str(num).zfill(5) + ".png"   # noqa: E731
    inputs = tuple(os.path.join(src, name(first + 8 * p)) for p in test_py_window(i, n))
    files = test_py_names(first + 8 * i)
    return WindowPaths(inputs, {k: os.path.join(gt_path, folder, f) for k, f in files.items()},
                       {k: os.path.join(gen_dir, folder, f) for k, f in files.items()},
                       os.path.join(src, name(first + 8 * min(i + 1, n - 1))))


def _scored(i: int, n: int) -> Tuple[int, ...]:
    """The pairs window i scores, in test.py's order (test.py:404-458): each written deblurred frame against its GT
    (12, then 8), the interpolated frame (13) and the blurry frame (-1) against the middle GT."""
    w = test_py_writes(i, n)
    return tuple(k for k in (12, 8) if k in w) + (13, -1)


# ----------------------------------------------------------------------------- logs (test.py:168-185, 404-506)
class AverageMeter:
    """utils/AverageMeter.py's arithmetic: sum += val * n; avg = sum / count."""

    def __init__(self):
        self.val = self.avg = self.sum = self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def _compare_psnr(s_sq: int, n: int):
    err = np.float64(s_sq / n)          # skimage compare_psnr on uint8 (metrics.compare_psnr)
    return np.float64(np.inf) if err == 0 else 10 * np.log10((255 ** 2) / err)


class Record(NamedTuple):
    folder: str
    i: int                              # window index
    h: int
    w: int
    rows: Tuple[Tuple[float, float, float, float], ...]   # per _scored pair: sum|a-b|, sum (a-b)^2, Gaussian, box SSIM


class Stopped(NamedTuple):
    folder: str
    i: int                              # the window whose interpolated frame equals its GT


def test_py_messages(header: Sequence[str], folders: Sequence[Tuple[str, int]], records: Sequence[Record],
                     model_size: str, runtime: float, blurry_path) -> Tuple[List[str], List[str], Optional[Stopped]]:
    """The messages test.py logs to test_*.log and test_summary_*.log, from the windows' metric sums.  folders: every
    (folder, frame count) in order; records: one per window (any order); blurry_path(folder, i): the path test.py logs
    after window i's blurry scores.  -> (log, summary, the window where test.py would have returned early, or None)."""
    log, summary = list(header), []
    at = {(r.folder, r.i): r for r in records}
    sets = collections.OrderedDict((k, AverageMeter()) for k in ("err", "pi", "si", "pd", "sd", "pb", "sb"))
    for folder, n in folders:
        m = {k: AverageMeter() for k in sets}
        log.append("The results for dir:{}".format(folder))
        summary.append("The results for dir:{}".format(folder))
        for i in range(max(n - 1, 0)):
            r = at[(folder, i)]
            px = r.h * r.w * 3
            rows = dict(zip(_scored(i, n), r.rows))
            for k in (12, 8):
                if k in rows:
                    psnr_tmp, ssim_tmp = _compare_psnr(int(rows[k][1]), px), np.float64(rows[k][3])
                    m["pd"].update(psnr_tmp, 1)
                    m["sd"].update(ssim_tmp, 1)
                    log.append("Interp PSNR : " + str(round(psnr_tmp, 4)) + " Interp SSIM : " + str(round(ssim_tmp, 4)))
            s_abs, s_sq, _, box = rows[13]
            avg_interp_error_abs = np.float64(int(s_abs) / px)
            m["err"].update(avg_interp_error_abs, 1)
            mse = np.float64(int(s_sq) / px)
            if mse == 0:
                return log, summary, Stopped(folder, i)
            psnr = 20 * math.log10(255.0 / math.sqrt(mse))
            m["pi"].update(psnr, 1)
            m["si"].update(np.float64(box), 1)
            log.append("deblur error / PSNR : " + str(round(avg_interp_error_abs, 4)) + " / " + str(round(psnr, 4)))
            psnr_tmp, ssim_tmp = _compare_psnr(int(rows[-1][1]), px), np.float64(rows[-1][3])
            m["pb"].update(psnr_tmp, 1)
            m["sb"].update(ssim_tmp, 1)
            log.append("blurry PSNR : " + str(round(psnr_tmp, 4)) + " blurry SSIM : " + str(round(ssim_tmp, 4)) + '\n'
                       + blurry_path(folder, i))
        summary.append("The results for dir:" + folder)
        summary.append("The average interpolation error " + str(round(m["err"].avg, 4)))
        summary.append("Avg. folder" + " blurry psnr " + str(m["pb"].avg) + " deblur psnr " + str(m["pi"].avg)
                       + " interp psnr " + str(m["pd"].avg) + " blurry ssim " + str(m["sb"].avg)
                       + " deblur ssim " + str(m["si"].avg) + " interp ssim " + str(m["sd"].avg))
        for k, s in sets.items():
            s.update(m[k].avg, 1)
    summary.append("The results for Adobe dataset")
    summary.append("The average interpolation error " + str(round(sets["err"].avg, 4)))
    summary.append("Avg. testset " + " interp psnr " + str(sets["pd"].avg) + " blurry psnr" + str(sets["pb"].avg)
                   + " deblur psnr" + str(sets["pi"].avg) + " interp ssim " + str(sets["sd"].avg)
                   + " blurry ssim" + str(sets["sb"].avg) + " deblur ssim" + str(sets["si"].avg))
    summary.append("runtime per image [s] : %.4f\n" % runtime + "CPU[1] / GPU[0] : 1 \n"
                   + "Extra Data [1] / No Extra Data [0] : 1")
    summary.append(model_size)
    return log, summary, None


def _write_log(path: str, messages: Sequence[str]) -> None:
    """The messages as utils/util.py:77-91 setup_logger's file handler formats them."""
    lg = logging.Logger(path, logging.INFO)         # not registered: repeated calls add no handlers to a shared logger
    fh = logging.FileHandler(path, mode="w")
    fh.setFormatter(logging.Formatter('%(asctime)s.%(msecs)03d - %(levelname)s: %(message)s', datefmt='%y-%m-%d %H:%M:%S'))
    lg.addHandler(fh)
    try:
        for msg in messages:
            lg.info(msg)
    finally:
        fh.close()


# ----------------------------------------------------------------------------- decoding
class _Prefetch:
    """cv2.imread of `paths` in order on `threads` host threads, each image copied into pinned memory, at most `depth`
    ahead of the consumer."""

    def __init__(self, paths: Sequence[str], threads: int, depth: int):
        self._paths = iter(paths)
        self._pool = cf.ThreadPoolExecutor(max(threads, 1), thread_name_prefix="bin_b200-decode")
        self._q: collections.deque = collections.deque()
        for _ in range(max(depth, 1)):
            self._submit()

    @staticmethod
    def _read(path: str) -> torch.Tensor:
        import cv2
        img = cv2.imread(path)
        if img is None:
            raise BinB200Error(f"evaluate_testset: cannot read {path}")
        return torch.from_numpy(img).pin_memory()

    def _submit(self):
        p = next(self._paths, None)
        if p is not None:
            self._q.append((p, self._pool.submit(self._read, p)))

    def get(self, path: str) -> torch.Tensor:
        p, fut = self._q.popleft()
        assert p == path, (p, path)             # the schedule and the consumer walk the same order
        self._submit()
        return fut.result()

    def close(self):
        for _, fut in self._q:
            fut.cancel()
        self._pool.shutdown(wait=True)


# ----------------------------------------------------------------------------- one rank's windows
def _folder_info(input_path: str, folder: str) -> Tuple[int, int]:
    """-> (frame count, first frame number) of a folder (test.py:244, 251-252); the names must run 8 apart."""
    names = sorted(os.listdir(os.path.join(input_path, folder)))
    if not names:
        return 0, 0
    first = int(names[0][:-4])
    want = [str(first + 8 * k).zfill(5) + ".png" for k in range(len(names))]
    if names != want:
        raise BinB200Error(f"evaluate_testset: the blurry frames of {folder} must be named {want[0]}, {want[1:2]}... 8 "
                           "apart (test.py:262-287 names its inputs that way)")
    return len(names), first


def _schedule(folder_n: int, rng: range) -> List[Tuple[str, object]]:
    """The order the rank consumes files in: frame p as it arrives, then the GTs of the windows due at it."""
    plan = VideoPlan(frozenset(), rng, folder_n)
    out = []
    while not plan.complete:
        pos = plan.next_pos
        out.append(("frame", pos))
        for step in plan.arrive():
            out += [("gt", (step.i, k)) for k in (12, 8, 13) if k in test_py_writes(step.i, folder_n)]
    return out


def _evaluate_rank(win_net, dev, pieces, info, input_path, gt_path, gen_dir, direct_interp, threads):
    """Run one rank's (folder, window range) pieces -> (records, seconds)."""
    sched = []                                      # (folder, kind, key, path)
    for folder, rng in pieces:
        n, first = info[folder]
        wp = lambda i: window_paths(input_path, gt_path, gen_dir, folder, first, i, n, direct_interp)   # noqa: E731
        for kind, key in _schedule(n, rng):
            if kind == "frame":
                p = os.path.join(gt_path if direct_interp else input_path, folder, str(first + 8 * key).zfill(5) + ".png")
            else:
                p = wp(key[0]).gt[key[1]]
            sched.append((folder, kind, key, p))
    pre = _Prefetch([s[3] for s in sched], threads, 4 * threads + 8)
    writer = cf.ThreadPoolExecutor(1, thread_name_prefix="bin_b200-write")
    writes: List[cf.Future] = []
    records: List[Record] = []
    pending = None
    cursor = iter(sched)

    def take(kind, key):
        _, k, kk, p = next(cursor)
        assert (k, kk) == (kind, key), ((k, kk), (kind, key))
        return pre.get(p)

    def finish(job):
        folder, i, hw, ev, host, png, paths = job
        for path, data in zip(paths, png.result()):
            writes.append(writer.submit(_write_file, path, data))
        ev.synchronize()
        records.append(Record(folder, i, hw[0], hw[1], tuple(tuple(r) for r in host.tolist())))

    t0 = time.perf_counter()
    try:
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream()
            for folder, rng in pieces:
                n, first = info[folder]
                blurry: Dict[int, torch.Tensor] = {}
                shape = {}

                def frames():
                    for pos in range(max(rng.start - 2, 0), min(rng.stop + 2, n - 1) + 1):
                        u8 = take("frame", pos).to(dev, non_blocking=True)
                        if not shape:
                            shape["hw"] = tuple(u8.shape[:2])
                            shape["pad"] = test_py_padding(*shape["hw"])
                        elif tuple(u8.shape[:2]) != shape["hw"]:
                            raise BinB200Error(f"evaluate_testset: the frames of {folder} differ in size")
                        blurry[pos] = u8
                        yield upload_frame_u8(u8, shape["pad"], dev)

                for i, outs in stream_video(win_net, frames(), windows=rng, n=n):
                    (h, w), (pl, _, pt, _) = shape["hw"], shape["pad"]
                    wp = window_paths(input_path, gt_path, gen_dir, folder, first, i, n, direct_interp)
                    todo = test_py_writes(i, n)
                    imgs = {k: tensor2img_u8(outs[k], crop=(pt, pl, h, w)) for k in todo}
                    gts = {}
                    for k in (12, 8, 13):
                        if k in todo:
                            gts[k] = take("gt", (i, k)).to(dev, non_blocking=True)
                            if tuple(gts[k].shape[:2]) != (h, w):
                                raise BinB200Error(f"evaluate_testset: {wp.gt[k]} is not {h}x{w}")
                    blur = blurry[min(i + 1, n - 1)]
                    pairs = [(imgs[k], gts[k]) if k >= 0 else (blur, gts[13]) for k in _scored(i, n)]
                    sums = image_metrics_batch(pairs, bgr=True)
                    host = torch.empty(sums.shape, dtype=torch.float64, pin_memory=True)
                    host.copy_(sums, non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(stream)
                    png = encode_png_async([imgs[k] for k in todo])
                    for p in [p for p in blurry if p < min(i + 1, n - 1)]:
                        del blurry[p]
                    if pending is not None:
                        finish(pending)             # window i-1's files and sums, while window i runs
                    pending = (folder, i, (h, w), ev, host, png, [wp.out[k] for k in todo])
            if pending is not None:
                finish(pending)
            for f in writes:
                f.result()
            torch.cuda.synchronize(dev)
    finally:
        pre.close()
        writer.shutdown(wait=True)
    return records, time.perf_counter() - t0


def _write_file(path: str, data: bytes) -> None:
    with open(path, "wb") as fh:
        fh.write(data)


def _gather(local, world: int) -> list:
    """Every rank's `local`, in rank order (torch.distributed when world > 1)."""
    if world == 1:
        return [local]
    out = [None] * world
    torch.distributed.all_gather_object(out, local)
    return out


def _window_net(net):
    nets = [m for m in net.modules() if isinstance(m, rdn.RDN_residual_interp_5_input_ConvLSTM_L)]
    if not nets:
        raise BinB200Error("evaluate_testset: no RDN_residual_interp_5_input_ConvLSTM_L in this module")
    return nets


def evaluate_testset(net, input_path: str, gt_path: str, output_path: str, net_name: str, *, direct_interp: bool = False,
                     rank: Optional[int] = None, world: Optional[int] = None, decode_threads: int = 8,
                     model_path: str = "") -> Optional[str]:
    """test.py's evaluation of a test set (test.py:73-506): the blurry frames under input_path/<folder>/, GT frames at
    240 fps names under gt_path/<folder>/, images written to output_path/60fps_test_results/<net_name>/<folder>/ and
    the logs test_<timestamp>.log and test_summary_<timestamp>.log beside them, with test.py's messages ("Model path:
    Joint Model:<model_path>"; only "runtime per image" holds this run's own time: seconds of evaluation per window,
    summed over the ranks).  net: a BIN window net, or a module holding one, on the device it runs on; it computes only
    (13, 8, 12) during the call, in its precision and self-ensemble modes ("Flip test: True" with flip-x4).

    rank / world default to the initialised process group, else (0, 1).  Each rank runs its contiguous run of windows
    (dist.shard_test_set) and writes its images; rank 0 writes the logs from the gathered records.  Raises
    BinB200Error if an image it would write exists, and where test.py returns early (an interpolated frame equal to its
    GT), after writing the logs up to that point.  -> the summary log's path on rank 0, else None."""
    if rank is None or world is None:
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            rank, world = torch.distributed.get_rank(), torch.distributed.get_world_size()
        else:
            rank, world = 0, 1
    if not 0 <= rank < world:
        raise BinB200Error(f"evaluate_testset: rank {rank} is not in 0..{world - 1}")
    nets = _window_net(net)
    dev = next(net.parameters()).device
    flip_test = rdn._ensemble_of(nets[0]) is not None
    result_path = os.path.join(output_path, RESULT_DIR)
    gen_dir = os.path.join(result_path, net_name)
    subdir = sorted(os.listdir(input_path))                                      # test.py:158
    info = {f: _folder_info(input_path, f) for f in subdir}
    pieces = bdist.shard_test_set({f: info[f][0] for f in subdir}, world)[rank]
    for f in subdir:
        os.makedirs(os.path.join(gen_dir, f), exist_ok=True)
    for folder, rng in pieces:
        n, first = info[folder]
        for i in rng:
            wp = window_paths(input_path, gt_path, gen_dir, folder, first, i, n, direct_interp)
            for k in test_py_writes(i, n):
                if os.path.exists(wp.out[k]):
                    raise BinB200Error(f"evaluate_testset: {wp.out[k]} exists; test.py would skip it and log other "
                                       "metrics, so evaluate into a directory without its images")

    saved = [getattr(m, "outputs", None) for m in nets]
    for m in nets:
        rdn.set_outputs(m, WANTED)
    try:
        records, seconds = _evaluate_rank(nets[0], dev, pieces, info, input_path, gt_path, gen_dir, direct_interp,
                                          decode_threads)
    finally:
        for m, sel in zip(nets, saved):
            m.outputs = sel
    ranks = _gather((records, seconds), world)
    all_records = [r for recs, _ in ranks for r in recs]
    nwin = len(all_records)
    runtime = sum(s for _, s in ranks) / nwin if nwin else 0.0
    n_params = sum([np.prod(p.size()) for p in net.parameters() if p.requires_grad])     # test.py:68-71
    model_size = 'Num. of model parameters is : {}'.format(str(n_params))
    header = ['In Data: {} '.format(input_path), 'Padding mode: {}'.format(PAD),
              'Model path: {}'.format("Joint Model:" + model_path), 'Save images: {}'.format(result_path),
              'Flip test: {}'.format(flip_test), 'Use ssin method {}'.format(SSIM_MSG), model_size]
    folders = [(f, info[f][0]) for f in subdir]

    def blurry_path(folder, i):
        return window_paths(input_path, gt_path, gen_dir, folder, info[folder][1], i, info[folder][0], direct_interp).blurry

    log, summary, stopped = test_py_messages(header, folders, all_records, model_size, runtime, blurry_path)
    summary_path = None
    if rank == 0:
        stamp = datetime.now().strftime('%y%m%d-%H%M%S')                        # utils/util.py:43-44
        _write_log(os.path.join(gen_dir, "test_{}.log".format(stamp)), log)
        summary_path = os.path.join(gen_dir, "test_summary_{}.log".format(stamp))
        _write_log(summary_path, summary)
    if stopped is not None:
        n, first = info[stopped.folder]
        path = window_paths(input_path, gt_path, gen_dir, stopped.folder, first, stopped.i, n, direct_interp).out[13]
        raise BinB200Error(f"evaluate_testset: {path} equals its GT (mse 0); test.py:440-441 returns here without a "
                           "summary, and the logs stop at the same message")
    return summary_path


# ----------------------------------------------------------------------------- command line
def _flag(v: str) -> bool:
    if v.lower() in ("1", "true", "yes", "on"):
        return True
    if v.lower() in ("", "0", "false", "no", "off"):
        return False
    raise argparse.ArgumentTypeError(f"not a truth value: {v!r}")


def load_weights(net, path: str) -> None:
    """base_model.load_network (base_model.py:89-103): the checkpoint's keys without their 'InterpNet.' / 'module.'
    prefix, loaded with strict=True."""
    sd = torch.load(path, map_location="cpu")
    clean = collections.OrderedDict()
    for k, v in sd.items():
        for pre in ("module.", "InterpNet."):
            if k.startswith(pre):
                k = k[len(pre):]
        clean[k] = v
    net.load_state_dict(clean, strict=True)


def main(argv=None) -> None:
    ap = argparse.ArgumentParser(description="test.py's test-set evaluation on the GPU (one process per GPU under "
                                             "torchrun)")
    ap.add_argument("--netName", required=True)
    ap.add_argument("--input_path", required=True)
    ap.add_argument("--gt_path", required=True)
    ap.add_argument("--output_path", required=True)
    ap.add_argument("--direct_interp", type=_flag, nargs="?", const=True, default=False)
    ap.add_argument("--weights", required=True, help="a bin_stage4 checkpoint, e.g. adobe_bin.pth")
    ap.add_argument("--precision", choices=("fp16", "fp32"), default="fp16")
    ap.add_argument("--flipx4", action="store_true", help="x4 flip self-ensemble (logged as 'Flip test: True')")
    ap.add_argument("--decode_threads", type=int, default=8)
    args = ap.parse_args(argv)

    distributed = int(os.environ.get("WORLD_SIZE", "1")) > 1
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if distributed:
        torch.distributed.init_process_group("nccl")
    try:
        net = rdn.bin_stage4_lstm()
        load_weights(net, args.weights)
        net = net.to(f"cuda:{local}").eval()
        bdist.broadcast_weights(net)
        rdn.set_precision(net, args.precision)
        rdn.set_self_ensemble(net, "flipx4" if args.flipx4 else None)
        path = evaluate_testset(net, args.input_path, args.gt_path, args.output_path, args.netName,
                                direct_interp=args.direct_interp, decode_threads=args.decode_threads,
                                model_path=args.weights)
        if path is not None:
            print(path)
    finally:
        if distributed:
            torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
