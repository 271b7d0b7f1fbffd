"""Blur synthesis for training data (SURVEY 8f rank 4): data_scripts/adobe240fps/create_dataset_blur_N_frames_average.py.

The script slides a window over the 240-fps sharp frames of one video (:99-140): blurry frame w is the float32 mean of
the `window_size` frames centred on `16 + 8*w`, truncated to uint8 (:117-131).  `blur_average` does every window of a
clip in one sm_90a launch on uint8 frames already in HBM, bit-exactly.  CUDA only; there is no CPU path."""
from __future__ import annotations

import math

import torch

from ._lib import BinB200Error, check, lib

WINDOW_MIDDLE = 16            # script :99  blurry_frame_idx = [16] (0-based; file name is idx+1)
WINDOW_MIDDLE_DELTA = 8       # script :103


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
