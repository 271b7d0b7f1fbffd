"""The blurred Adobe240 dataset (SURVEY 8f rank 4): data_scripts/adobe240fps/create_dataset_blur_N_frames_average.py.

The script slides a window over the 240-fps sharp frames of one video (:99-140): blurry frame w is the float32 mean of
the `window_size` frames centred on `16 + 8*w`, truncated to uint8 (:117-131).  `blur_average` does every window of a
clip in one sm_90a launch on uint8 frames already in HBM, bit-exactly.  CUDA only; there is no CPU path.

`build_dataset` (and ``python -m bin_b200.dataprep``, which takes the script's arguments) writes the tree the script
writes, video by video in its order: extract the frames with ffmpeg into `full_sharp/<stem>` unless that folder exists
(:36-67), write `<split>_blur/<stem>/NNNNN.png` (:86-140), copy `full_sharp/<stem>` to `<split>/<stem>` unless it
exists (:142-143) and write `<split>_list/<stem>_im_list.txt` (:145-148).  Each sharp frame is decoded once, with cv2
on host threads; windows are averaged on the device CHUNK_WINDOWS at a time and encoded by the GPU PNG encoder, and a
host thread writes each chunk's files while the next chunk runs.  The pixels are the script's; the PNG bytes are not
PIL's (the deflate differs).  Where this departs from the script:

  * a non-zero ffmpeg exit raises (and removes the folder it was extracting into), where the script prints and goes on;
  * without `ffmpeg_dir` every `full_sharp/<stem>` must exist;
  * the frame names must run 00001.png, 00002.png, ... with no gap (the script asserts only the first, and a gap shifts
    its windows), frames must be 8-bit 3-channel and of one size, and a window that reads outside the frames is refused
    before anything of that video is written (the script dies in imread);
  * empty lines of a video list are skipped (the script reads one as a video named '' and fails);
  * the custom-dataset branch (:203-226) is refused: it calls create_clips_overlap with two of its five arguments."""
from __future__ import annotations

import argparse
import concurrent.futures as cf
import math
import os
import shutil
import subprocess
from typing import List, NamedTuple, Optional, Tuple

import numpy as np
import torch

from ._lib import BinB200Error, check, lib

WINDOW_MIDDLE = 16            # script :99  blurry_frame_idx = [16] (0-based; file name is idx+1)
WINDOW_MIDDLE_DELTA = 8       # script :103
DATASETS = ("adobe240fps_blur", "youtube240fps_blur")     # script :179
CHUNK_WINDOWS = 16            # windows per device chunk: 131 frames at window_size 11, 362 MB at 1280x720


def window_count(n_frames: int) -> int:
    """script :104  window_total_num = floor(n_length / window_middle_delta) - 2"""
    return math.floor(n_frames / WINDOW_MIDDLE_DELTA) - 2


def blur_average(frames: torch.Tensor, window_size: int = 11, first_mid: int = WINDOW_MIDDLE,
                 stride: int = WINDOW_MIDDLE_DELTA, nwin: int | None = None) -> torch.Tensor:
    """frames: uint8 CUDA tensor (T, ...) of consecutive sharp frames -> uint8 (nwin, ...) blurry frames."""
    if not (frames.is_cuda and frames.dtype == torch.uint8):
        raise BinB200Error("blur_average: uint8 CUDA frames only (no CPU path)")
    frames = frames.contiguous()
    T = frames.shape[0]
    if nwin is None:
        nwin = window_count(T)
    if nwin < 1:
        raise BinB200Error(f"blur_average: {T} frames hold no complete window")
    frame_bytes = frames[0].numel()
    out = torch.empty((nwin,) + tuple(frames.shape[1:]), dtype=torch.uint8, device=frames.device)
    with torch.cuda.device(frames.device):
        check(lib().bin_blur_average_u8(frames.data_ptr(), T, frame_bytes, window_size, first_mid, stride, nwin,
                                        out.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return out


# ----------------------------------------------------------------------------- the script's steps
def frame_name(k: int) -> str:
    """The file of 0-based frame k (script :124): ffmpeg's %05d numbering from 1."""
    return str(k + 1).zfill(5) + ".png"


def ffmpeg_argv(ffmpeg_dir: str, videos_folder: str, video: str, out_dir: str, img_width: int,
                img_height: int) -> List[str]:
    """The command of script :59-65, one argument per word of its shell string."""
    return [os.path.join(ffmpeg_dir, "ffmpeg"), "-i", os.path.join(videos_folder, video), "-vf",
            "scale={}:{}".format(img_width, img_height), "-vsync", "0", "-qscale:v", "2", "{}/%05d.png".format(out_dir)]


def extract_frames(video: str, videos_folder: str, extract_root: str, ffmpeg_dir: str, img_width: int,
                   img_height: int) -> bool:
    """script :54-67 for one video: run ffmpeg into extract_root/<stem> unless that folder exists.  -> whether ffmpeg
    ran.  A non-zero exit removes the folder (so the next run extracts again) and raises."""
    out_dir = os.path.join(extract_root, os.path.splitext(video)[0])
    if os.path.exists(out_dir):
        return False
    os.makedirs(out_dir, exist_ok=True)
    argv = ffmpeg_argv(ffmpeg_dir, videos_folder, video, out_dir, img_width, img_height)
    try:
        code = subprocess.run(argv).returncode
    except OSError as e:
        code = e
    if code != 0:
        shutil.rmtree(out_dir, ignore_errors=True)
        raise BinB200Error(f"build_dataset: ffmpeg failed on {video} ({code}): {' '.join(argv)}")
    return True


def frame_count(folder: str) -> int:
    """The number of frames of an extracted folder, whose names must be exactly 00001.png .. NNNNN.png."""
    names = sorted(os.listdir(folder))
    if not names:
        raise BinB200Error(f"build_dataset: {folder} holds no frames")
    for k, n in enumerate(names):
        if n != frame_name(k):
            raise BinB200Error(f"build_dataset: {folder} must hold 00001.png ... {frame_name(len(names) - 1)} with no "
                               f"gap; found {n} where {frame_name(k)} belongs")
    return len(names)


def window_mids(n_frames: int, window_size: int, folder: str = "") -> List[int]:
    """The 0-based middle frame of each window (script :99-139): 16 + 8w for floor(T/8) - 2 windows, each averaging
    the 2r + 1 frames mid - r .. mid + r, r = int((window_size - 1) / 2).  Raises if a window reads outside the frames."""
    r = int((window_size - 1) / 2)
    mids = [WINDOW_MIDDLE + WINDOW_MIDDLE_DELTA * w for w in range(max(window_count(n_frames), 0))]
    if mids and (mids[0] - r < 0 or mids[-1] + r >= n_frames):
        raise BinB200Error(f"build_dataset: window_size {window_size} reads frames {mids[0] - r + 1}..{mids[-1] + r + 1} "
                           f"of {folder or 'a video'}, which has {n_frames}")
    return mids


def read_frame(path: str) -> np.ndarray:
    """cv2.imread(IMREAD_UNCHANGED) of one sharp frame, which must be 8-bit with 3 channels: (h, w, 3) BGR."""
    import cv2
    img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if img is None:
        raise BinB200Error(f"build_dataset: cannot read {path}")
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
        raise BinB200Error(f"build_dataset: {path} is not an 8-bit 3-channel image ({img.dtype}, shape "
                           f"{tuple(img.shape)})")
    return img


def read_video_list(path: str) -> List[str]:
    """script :180-184, 192-193: one video file name per line; empty lines are skipped."""
    if not os.path.isfile(path):
        raise BinB200Error(f"build_dataset: video list {path} does not exist")
    with open(path) as fh:
        return [v for v in fh.read().split("\n") if v]


def chunks(mids: List[int], window_size: int, per_chunk: int) -> List[Tuple[List[int], int, int]]:
    """The device chunks of a video's windows: (the middles of up to per_chunk consecutive windows, the first and the
    last frame they read)."""
    r = int((window_size - 1) / 2)
    return [(mids[i:i + per_chunk], mids[i] - r, mids[min(i + per_chunk, len(mids)) - 1] + r)
            for i in range(0, len(mids), per_chunk)]


def blur_video(src: str, dst: str, mids: List[int], window_size: int, device, threads: int = 8) -> List[str]:
    """script :108-134 for one video: the blurry frame of every window in `mids` from the frames in src, written to
    dst/<name of the middle frame>.  Frames are decoded once each on `threads` host threads; CHUNK_WINDOWS windows are
    uploaded, averaged and encoded at a time, and one chunk's files are written while the next chunk runs.
    -> the names written, in order."""
    from .evaluate import _Prefetch, _write_file
    from .png import encode_png_async
    if not mids:
        return []
    if not torch.cuda.is_available():
        raise BinB200Error("build_dataset: no CUDA device (bin_b200 has no CPU path)")
    r = int((window_size - 1) / 2)
    needed = sorted({k for m in mids for k in range(m - r, m + r + 1)})
    os.makedirs(dst, exist_ok=True)
    dev = torch.device(device)
    pre = _Prefetch([os.path.join(src, frame_name(k)) for k in needed], threads, 4 * threads + 8, "build_dataset",
                    read=read_frame)
    writer = cf.ThreadPoolExecutor(1, thread_name_prefix="bin_b200-write")
    writes: List[cf.Future] = []
    held = {}                                   # frame -> pinned host image, while a later chunk still reads it
    shape = None
    pending = None
    at = 0                                      # next index into `needed`

    def finish(job):
        png, names = job
        for name, data in zip(names, png.result()):
            writes.append(writer.submit(_write_file, os.path.join(dst, name), data))

    try:
        with torch.cuda.device(dev):
            for chunk, lo, hi in chunks(mids, window_size, CHUNK_WINDOWS):
                while at < len(needed) and needed[at] <= hi:
                    k = needed[at]
                    img = pre.get(os.path.join(src, frame_name(k)))
                    if shape is None:
                        shape = tuple(img.shape)
                    elif tuple(img.shape) != shape:
                        raise BinB200Error(f"build_dataset: {os.path.join(src, frame_name(k))} is "
                                           f"{tuple(img.shape)}, the frames before it {shape}")
                    held[k] = img
                    at += 1
                for k in [k for k in held if k < lo]:
                    del held[k]
                # frames between windows (window_size < 9) are read by no window and stay unset
                frames = torch.empty((hi - lo + 1,) + shape, dtype=torch.uint8, device=dev)
                for k, img in held.items():
                    frames[k - lo].copy_(img, non_blocking=True)
                out = blur_average(frames, window_size, first_mid=chunk[0] - lo, nwin=len(chunk))
                png = encode_png_async(list(out.unbind(0)))
                if pending is not None:
                    finish(pending)             # the previous chunk's files, while this one runs
                pending = (png, [frame_name(m) for m in chunk])
            finish(pending)
            for f in writes:
                f.result()
    finally:
        pre.close()
        writer.shutdown(wait=True)
    return [frame_name(m) for m in mids]


class VideoDone(NamedTuple):
    split: str                  # "test" or "train"
    stem: str
    frames: int                 # sharp frames
    blurry: int                 # blurry frames written
    extracted: bool             # ffmpeg ran
    copied: bool                # the sharp frames were copied to <split>/<stem>


def build_dataset(dataset_folder: str, *, test_list: str = "./test_list.txt", train_list: Optional[str] = None,
                  videos_folder: Optional[str] = None, ffmpeg_dir: Optional[str] = None, img_width: int = 256,
                  img_height: int = 128, window_size: int = 7, enable_train: int = 0,
                  dataset: str = "adobe240fps_blur", decode_threads: int = 8, device="cuda") -> List[VideoDone]:
    """create_dataset_blur_N_frames_average.py's main() (:152-199) with its defaults: the videos of test_list, then
    with enable_train == 1 those of train_list (default `<dataset without _blur>/train_list.txt`, as the script), each
    extracted, blurred, copied and listed in turn under dataset_folder.  The lists, the dataset, window_size and (without
    ffmpeg_dir) every full_sharp/<stem> are checked before any video is processed.  -> one VideoDone per video."""
    if dataset not in DATASETS:
        raise BinB200Error(f"build_dataset: dataset must be one of {DATASETS}, got {dataset!r}; the script's custom-"
                           "dataset branch calls create_clips_overlap with two of its five arguments, so it cannot run")
    if not 1 <= window_size <= 256:
        raise BinB200Error(f"build_dataset: window_size must be in 1..256, got {window_size}")
    if ffmpeg_dir is not None and videos_folder is None:
        raise BinB200Error("build_dataset: ffmpeg_dir needs videos_folder")
    if train_list is None:
        train_list = dataset[:-5] + "/train_list.txt"
    splits = [("test", read_video_list(test_list))]
    if enable_train == 1:
        splits.append(("train", read_video_list(train_list)))
    extract_root = os.path.join(dataset_folder, "full_sharp")
    if ffmpeg_dir is None:
        for _, videos in splits:
            for v in videos:
                if not os.path.isdir(os.path.join(extract_root, os.path.splitext(v)[0])):
                    raise BinB200Error(f"build_dataset: {os.path.join(extract_root, os.path.splitext(v)[0])} does not "
                                       "exist; extract the frames of " f"{v} there or give ffmpeg_dir")
    for sub in ("full_sharp", "train", "test", "train_list", "test_list", "train_blur", "test_blur"):    # :170-177
        os.makedirs(os.path.join(dataset_folder, sub), exist_ok=True)
    done = []
    for split, videos in splits:
        for video in videos:
            stem = os.path.splitext(video)[0]
            src = os.path.join(extract_root, stem)
            extracted = ffmpeg_dir is not None and extract_frames(video, videos_folder, extract_root, ffmpeg_dir,
                                                                  img_width, img_height)
            T = frame_count(src)
            mids = window_mids(T, window_size, src)
            names = blur_video(src, os.path.join(dataset_folder, split + "_blur", stem), mids, window_size, device,
                               decode_threads)
            dst = os.path.join(dataset_folder, split, stem)
            copied = not os.path.exists(dst)
            if copied:
                shutil.copytree(src, dst)
            with open(os.path.join(dataset_folder, split + "_list", stem + "_im_list.txt"), "w") as fh:
                fh.write("\n".join(names))                               # :145-148, no trailing newline
            print(f"{split} {stem}: {T} frames -> {len(names)} blurry frames", flush=True)
            done.append(VideoDone(split, stem, T, len(names), extracted, copied))
    return done


def parse_args(argv=None) -> argparse.Namespace:
    """The script's arguments (:21-31) and defaults, without --train_test_split (custom datasets only), plus the video
    lists the script opens from the working directory and the decode thread count."""
    ap = argparse.ArgumentParser(description="create_dataset_blur_N_frames_average.py on the GPU: the blurred "
                                             "Adobe240 tree (test_blur, test, test_list, train_blur, train, train_list)")
    ap.add_argument("--ffmpeg_dir", type=str, default=None,
                    help="folder holding ffmpeg; without it every <dataset_folder>/full_sharp/<stem> must exist")
    ap.add_argument("--dataset", type=str, default="adobe240fps_blur", help="adobe240fps_blur or youtube240fps_blur")
    ap.add_argument("--videos_folder", type=str, default=None, help="folder holding the videos (with --ffmpeg_dir)")
    ap.add_argument("--dataset_folder", type=str, required=True, help="the output tree")
    ap.add_argument("--img_width", type=int, default=256)
    ap.add_argument("--img_height", type=int, default=128)
    ap.add_argument("--window_size", type=int, default=7, help="sharp frames averaged per blurry frame")
    ap.add_argument("--enable_train", type=int, default=0, help="1: also build the train split")
    ap.add_argument("--test_list", type=str, default="./test_list.txt", help="the test videos, one per line")
    ap.add_argument("--train_list", type=str, default=None,
                    help="the train videos, one per line (default <dataset without _blur>/train_list.txt)")
    ap.add_argument("--decode_threads", type=int, default=8)
    return ap.parse_args(argv)


def main(argv=None) -> None:
    args = parse_args(argv)
    build_dataset(args.dataset_folder, test_list=args.test_list, train_list=args.train_list,
                  videos_folder=args.videos_folder, ffmpeg_dir=args.ffmpeg_dir, img_width=args.img_width,
                  img_height=args.img_height, window_size=args.window_size, enable_train=args.enable_train,
                  dataset=args.dataset, decode_threads=args.decode_threads)


if __name__ == "__main__":
    main()
