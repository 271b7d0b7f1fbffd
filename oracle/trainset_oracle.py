"""NumPy restatement of the reference's training-set loader, for the tests (our own code, written from the behaviour the
reference documents and the fixture pins; nothing of the reference is copied):

* ``windows``: data/BIN_dataset.py:186-288 ``_make_dataset_deep_long_``.  Folders in the order given (the reference
  takes ``os.listdir``); ``first`` = integer name of the first blurry file; ``len(blurry) - 5`` windows; window j reads
  blurry / sharp files ``first + 8(j+k)`` (k < 6) and sharp files ``first + 8(j+k) + 4`` (k < 5); it is dropped unless
  its six blurry names are in the folder's im_list; key ``folder_zfill(first + 8j, 5)``; one ``rng.shuffle``.
* ``sample``: :62-183 ``Adobe_BIN_loader`` + :30-54 ``__getitem__``: draws ``randint(0, 1)`` (0 reverses the three
  lists), ``choice(range(352 - h + 1))``, ``choice(range(640 - w + 1))``, ``randint(0, 1)`` (1 = fliplr), in that
  order; ``uint8 / 255.`` in float32; crop; flip; BGR -> RGB; (n,3,h,w).

Frames are held as the library holds them: ``blurry[i]`` is file ``first + 8i`` and ``sharp[m]`` is file
``first + 4m`` (the only sharp files a window reads).  ``CLIPS`` / ``synth_clip`` define the synthetic tree of
tests/golden/trainset.npz (oracle/make_golden_trainset.py).
"""
from __future__ import annotations

import hashlib
import os
from typing import Dict, List, Sequence, Tuple

import numpy as np

from . import bin_oracle as O

CROP_H, CROP_W = 352, 640          # the loader's hard-coded crop range (:132-133)
N_LQ, N_ENH, N_INP = 6, 6, 5

# folder, sharp frames T, H, W, frame seed, blurry names left out of the folder's im_list
CLIPS = (
    ("GOPR0384_11_00", 72, 352, 640, 1101, ()),
    ("IMG_0030", 80, 352, 640, 1102, ("00017.png",)),     # drops window 0: the im_list filter
    ("GOPR0871_11_01", 72, 360, 656, 1103, ()),           # larger frames: only their top-left 352x640 is cropped
)
LQ_SIZES = {"a": (128, 256), "b": (127, 255), "c": (352, 640)}


def synth_clip(T: int, H: int, W: int, seed: int) -> np.ndarray:
    """(T,H,W,3) uint8 sharp frames; frame k is file k+1 as the blur script numbers them."""
    return np.random.default_rng(seed).integers(0, 256, size=(T, H, W, 3), dtype=np.uint8)


def clip_arrays(T: int, H: int, W: int, seed: int, window_size: int = 11):
    """-> (all sharp frames, blurry frames, kept sharp frames, first): the blurry frames of the blur script
    (bin_oracle.blur_average: file 17 + 8w is the mean around 0-based frame 16 + 8w) and the sharp frames 16 + 4m."""
    sharp = synth_clip(T, H, W, seed)
    blurry = O.blur_average(sharp, window_size=window_size)
    kept = sharp[16:16 + 4 * (2 * len(blurry) - 1):4]
    return sharp, blurry, kept, 17


def name(i: int) -> str:
    return str(i).zfill(5)


def windows(clips: Sequence[Dict], rng) -> List[Tuple[int, int, str]]:
    """clips: dicts with folder, first, nb (blurry count), im_list (set of names or None) -> shuffled
    [(clip index, window j, key)]."""
    out = []
    for ci, c in enumerate(clips):
        first = c["first"]
        for j in range(c["nb"] - 5):
            names = [name(first + 8 * (j + k)) + ".png" for k in range(N_LQ)]
            if c["im_list"] is None or all(n in c["im_list"] for n in names):
                out.append((ci, j, c["folder"] + "_" + name(first + 8 * j)))
    rng.shuffle(out)
    return out


def draw(rng, h: int, w: int) -> Tuple[int, int, int, int]:
    """(order, top, left, flip) in the loader's order of draws."""
    order = rng.randint(0, 1)
    top = rng.choice(range(CROP_H - h + 1))
    left = rng.choice(range(CROP_W - w + 1))
    flip = rng.randint(0, 1)
    return order, top, left, flip


def frame_lists(blurry: np.ndarray, kept: np.ndarray, j: int, order: int):
    """The (LQs, GTenh, GTinp) uint8 frame lists of window j after the order draw."""
    lq = [blurry[j + k] for k in range(N_LQ)]
    enh = [kept[2 * (j + k)] for k in range(N_ENH)]
    inp = [kept[2 * (j + k) + 1] for k in range(N_INP)]
    if not order:
        lq, enh, inp = lq[::-1], enh[::-1], inp[::-1]
    return lq, enh, inp


def crop_stack(frames: Sequence[np.ndarray], top: int, left: int, flip: int, h: int, w: int) -> np.ndarray:
    """read_img's float32 / 255., the crop, np.fliplr, BGR -> RGB, HWC -> CHW: (n,3,h,w) float32."""
    out = []
    for f in frames:
        x = f.astype(np.float32) / 255.
        x = x[top:top + h, left:left + w, :]
        if flip:
            x = np.fliplr(x)
        out.append(x[:, :, [2, 1, 0]])
    return np.ascontiguousarray(np.stack(out).transpose(0, 3, 1, 2))


def sample(blurry, kept, j: int, d: Tuple[int, int, int, int], h: int, w: int):
    """-> {'LQs', 'GTenh', 'GTinp'} float32 arrays of window j under draws d = (order, top, left, flip)."""
    order, top, left, flip = d
    lq, enh, inp = frame_lists(blurry, kept, j, order)
    return {"LQs": crop_stack(lq, top, left, flip, h, w), "GTenh": crop_stack(enh, top, left, flip, h, w),
            "GTinp": crop_stack(inp, top, left, flip, h, w)}


def sha256(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def write_tree(root: str, clips=CLIPS, mode: str = "train") -> None:
    """The directory layout the reference reads: mode/<folder>/NNNNN.png (every sharp frame, 1-based),
    mode_blur/<folder>/NNNNN.png (blurry frame 17 + 8w), mode_list/<folder>_im_list.txt."""
    import cv2
    os.makedirs(os.path.join(root, mode + "_list"), exist_ok=True)
    for folder, T, H, W, seed, omit in clips:
        sharp, blurry, _, first = clip_arrays(T, H, W, seed)
        for sub, frames, names in ((mode, sharp, [name(k + 1) for k in range(T)]),
                                   (mode + "_blur", blurry, [name(first + 8 * i) for i in range(len(blurry))])):
            os.makedirs(os.path.join(root, sub, folder), exist_ok=True)
            for f, n in zip(frames, names):
                assert cv2.imwrite(os.path.join(root, sub, folder, n + ".png"), f)
        listed = [name(first + 8 * i) + ".png" for i in range(len(blurry))]
        with open(os.path.join(root, mode + "_list", folder + "_im_list.txt"), "w") as fh:
            fh.write("\n".join(n for n in listed if n not in omit))
