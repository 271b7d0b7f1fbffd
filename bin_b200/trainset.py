"""Training batches built on the GPU from clips held in HBM: data/BIN_dataset.py BINDataset + the DataLoader collation
of data/__init__.py create_dataloader, bit for bit.

The reference decodes 17 PNGs per sample and crops, flips, reorders and converts them in NumPy on the CPU.  Here every
clip is uploaded once as uint8; a batch is then one `bin_train_batch_u8` launch per 16 samples that reads the crops
straight from those frames.  The windows, keys, shuffle and per-sample draws are the reference's, made with the same
`random` calls in the same order, so `random.seed(s)` gives the same batches.  CUDA only; there is no CPU path."""
from __future__ import annotations

import os
import random
from concurrent.futures import ThreadPoolExecutor
from typing import Dict, Iterable, Iterator, List, Optional, Sequence, Tuple

import torch

from . import ops
from ._lib import BinB200Error
from .dataprep import blur_average

CROP_H, CROP_W = 352, 640          # BIN_dataset.py:132-133 draw the crop inside the top-left 352x640 of any frame
N_LQ, N_ENH, N_INP = 6, 6, 5       # 17 frames per sample: blurry, sharp ("GTenh") and in-between sharp ("GTinp")


def _name(i: int) -> str:
    return str(i).zfill(5)


def _windows(folder: str, first: int, nb: int, im_list: Optional[set]) -> List[Tuple[int, str]]:
    out = []
    for j in range(nb - 5):
        names = [_name(first + 8 * (j + k)) + ".png" for k in range(N_LQ)]
        if im_list is None or all(n in im_list for n in names):
            out.append((j, folder + "_" + _name(first + 8 * j)))
    return out


class DeviceClip:
    """One folder of the training set, on the device.

    blurry_u8: uint8 CUDA (nb,H,W,3) BGR frames; blurry_u8[i] is blurry file `first_index + 8i`.
    sharp_u8:  uint8 CUDA (ns,H,W,3) BGR frames; sharp_u8[m] is sharp file `first_index + 4m`.  These are the only sharp
               files a window reads (`first + 8(j+k)` and `first + 8(j+k) + 4`), so nb blurry frames need 2nb - 1.
    im_list:   the blurry file names of `<mode>_list/<folder>_im_list.txt`, or None for all of them."""

    def __init__(self, name: str, blurry_u8: torch.Tensor, sharp_u8: torch.Tensor, first_index: int = 17,
                 im_list: Optional[Iterable[str]] = None):
        for what, t in (("blurry_u8", blurry_u8), ("sharp_u8", sharp_u8)):
            if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8:
                raise BinB200Error(f"DeviceClip {name}: {what} must be a uint8 tensor")
            if t.dim() != 4 or t.shape[3] != 3 or t.shape[0] < 1:
                raise BinB200Error(f"DeviceClip {name}: {what} must be (n,H,W,3) BGR frames, got {tuple(t.shape)}")
        if blurry_u8.shape[1:] != sharp_u8.shape[1:]:
            raise BinB200Error(f"DeviceClip {name}: blurry {tuple(blurry_u8.shape)} and sharp {tuple(sharp_u8.shape)} "
                               "frames must share H and W")
        H, W = blurry_u8.shape[1], blurry_u8.shape[2]
        if H < CROP_H or W < CROP_W:
            raise BinB200Error(f"DeviceClip {name}: frames are {H}x{W}; the loader crops inside {CROP_H}x{CROP_W}")
        nb = blurry_u8.shape[0]
        if nb > 5 and sharp_u8.shape[0] < 2 * nb - 1:
            raise BinB200Error(f"DeviceClip {name}: {nb} blurry frames read {2 * nb - 1} sharp frames, got "
                               f"{sharp_u8.shape[0]}")
        if int(first_index) < 0:
            raise BinB200Error(f"DeviceClip {name}: first_index must be >= 0")
        if not (blurry_u8.is_cuda and sharp_u8.is_cuda) or blurry_u8.device != sharp_u8.device:
            raise BinB200Error(f"DeviceClip {name}: frames must be CUDA tensors on one device (no CPU path)")
        self.name, self.first = name, int(first_index)
        self.blurry, self.sharp = blurry_u8.contiguous(), sharp_u8.contiguous()
        self.im_list = None if im_list is None else set(im_list)
        self._blurry, self._sharp = self.blurry.unbind(0), self.sharp.unbind(0)

    @classmethod
    def from_sharp(cls, name: str, sharp_u8: torch.Tensor, window_size: int = 11,
                   im_list: Optional[Iterable[str]] = None) -> "DeviceClip":
        """A clip from all its sharp frames (T,H,W,3), 0-based frame k = file k+1: the blurry frames come from
        `dataprep.blur_average` (file 17 + 8w), and only the sharp frames 16 + 4m that a window reads are kept."""
        blurry = blur_average(sharp_u8, window_size=window_size)
        kept = sharp_u8[16:16 + 4 * (2 * blurry.shape[0] - 1):4].contiguous()
        return cls(name, blurry, kept, 17, im_list)

    def windows(self) -> List[Tuple[int, str]]:
        """(j, key) of every window the reference keeps, in its order (BIN_dataset.py:238-281)."""
        return _windows(self.name, self.first, self.blurry.shape[0], self.im_list)

    def frames(self, j: int, order: int) -> List[torch.Tensor]:
        """The 17 frames of window j in output order; order 0 reverses each of the three lists (BIN_dataset.py:68-109)."""
        lq = [self._blurry[j + k] for k in range(N_LQ)]
        enh = [self._sharp[2 * (j + k)] for k in range(N_ENH)]
        inp = [self._sharp[2 * (j + k) + 1] for k in range(N_INP)]
        if not order:
            lq, enh, inp = lq[::-1], enh[::-1], inp[::-1]
        return lq + enh + inp


class DeviceBINDataset:
    """BINDataset (data/BIN_dataset.py) over DeviceClips, with `keys`, `len()`, `ds[i]`, `batch` and `batches`.

    clips are taken in the order given (the reference takes `os.listdir(<root>/<mode>_blur)`); the window list is
    shuffled once with `rng.shuffle` at construction, and every sample makes the loader's four draws on `rng`
    (`random` by default, as the reference).  Parity holds for samples drawn in index order, as `n_workers: 0` does."""

    def __init__(self, clips: Sequence[DeviceClip], lq_size=(3, 128, 256), rng=random):
        h, w = int(lq_size[-2]), int(lq_size[-1])
        if not (1 <= h <= CROP_H and 1 <= w <= CROP_W):
            raise BinB200Error(f"DeviceBINDataset: lq_size {tuple(lq_size)} must crop inside {CROP_H}x{CROP_W}")
        if len({c.blurry.device for c in clips}) > 1:
            raise BinB200Error("DeviceBINDataset: all clips must be on one device")
        self.clips, self.h, self.w, self.rng = list(clips), h, w, rng
        self._win = [(c, j, key) for c in self.clips for j, key in c.windows()]
        rng.shuffle(self._win)
        self.keys = [k for _, _, k in self._win]

    def __len__(self) -> int:
        return len(self._win)

    def _draw(self, i: int):
        clip, j, key = self._win[i]
        order = self.rng.randint(0, 1)
        top = self.rng.choice(range(CROP_H - self.h + 1))
        left = self.rng.choice(range(CROP_W - self.w + 1))
        flip = self.rng.randint(0, 1)
        return (clip.frames(j, order), top, left, flip), key

    def batch(self, indices: Sequence[int]) -> Dict:
        """default_collate of [ds[i] for i in indices], with the draws made in that order: 'LQs' (B,6,3,h,w), 'GTenh'
        (B,6,3,h,w), 'GTinp' (B,5,3,h,w) fp32 views of one (17,B,3,h,w) buffer, so `LQs[:, k]` is a contiguous
        (B,3,h,w) batch; 'key' a list of B strings."""
        if len(indices) < 1:
            raise BinB200Error("DeviceBINDataset.batch: no indices")
        drawn = [self._draw(i) for i in indices]
        buf = ops.train_batch_u8([s for s, _ in drawn], self.h, self.w)
        return {"LQs": buf[0:N_LQ].transpose(0, 1), "GTenh": buf[N_LQ:N_LQ + N_ENH].transpose(0, 1),
                "GTinp": buf[N_LQ + N_ENH:].transpose(0, 1), "key": [k for _, k in drawn]}

    def __getitem__(self, i: int) -> Dict:
        """BINDataset.__getitem__: (6,3,h,w), (6,3,h,w), (5,3,h,w) and the key."""
        b = self.batch([i])
        return {"LQs": b["LQs"][0], "GTenh": b["GTenh"][0], "GTinp": b["GTinp"][0], "key": b["key"][0]}

    def batches(self, sampler: Iterable[int], batch_size: int) -> Iterator[Dict]:
        """DataLoader(batch_size, sampler, drop_last=True) over any iterable of indices (e.g. the reference's
        DistIterSampler)."""
        if batch_size < 1:
            raise BinB200Error("DeviceBINDataset.batches: batch_size must be >= 1")
        chunk = []
        for i in sampler:
            chunk.append(i)
            if len(chunk) == batch_size:
                yield self.batch(chunk)
                chunk = []

    @classmethod
    def from_tree(cls, root: str, mode: str = "train", folders: Optional[Sequence[str]] = None, device="cuda",
                  lq_size=(3, 128, 256), rng=random) -> "DeviceBINDataset":
        """The layout the reference reads: `<root>/<mode>/<folder>/NNNNN.png` (sharp), `<root>/<mode>_blur/<folder>`
        (blurry), `<root>/<mode>_list/<folder>_im_list.txt`; folders default to `os.listdir(<root>/<mode>_blur)`.
        PNGs are decoded as data/util.py read_img does (cv2.imread(IMREAD_UNCHANGED), first 3 channels) on host
        threads; only the files a kept window reads are decoded and uploaded (the rest of a clip tensor stays zero)."""
        import cv2
        if folders is None:
            folders = os.listdir(os.path.join(root, mode + "_blur"))
        dev = torch.device(device)

        def read(path):
            img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
            if img is None or img.dtype != "uint8" or img.ndim != 3 or img.shape[2] < 3:
                raise BinB200Error(f"from_tree: {path} is not an 8-bit colour image")
            return img[:, :, :3]

        def upload(pool, files, n):
            imgs = list(pool.map(read, [p for _, p in files]))
            if len({i.shape for i in imgs}) != 1:
                raise BinB200Error(f"from_tree: frames of different sizes {sorted({i.shape for i in imgs})}")
            out = torch.zeros((n,) + imgs[0].shape, dtype=torch.uint8, device=dev)
            for (k, _), img in zip(files, imgs):
                out[k].copy_(torch.from_numpy(img))
            return out

        clips = []
        with ThreadPoolExecutor(min(16, os.cpu_count() or 1)) as pool:
            for folder in folders:
                bdir, sdir = os.path.join(root, mode + "_blur", folder), os.path.join(root, mode, folder)
                bnames = sorted(os.listdir(bdir))
                first, nb = int(bnames[0][:-4]), len(bnames)
                with open(os.path.join(root, mode + "_list", folder + "_im_list.txt")) as fh:
                    im_list = set(fh.read().split("\n"))
                kept = [j for j, _ in _windows(folder, first, nb, im_list)]
                if not kept:
                    continue
                bidx = sorted({j + k for j in kept for k in range(N_LQ)})
                sidx = sorted({2 * (j + k) for j in kept for k in range(N_ENH)} |
                              {2 * (j + k) + 1 for j in kept for k in range(N_INP)})
                blurry = upload(pool, [(i, os.path.join(bdir, _name(first + 8 * i) + ".png")) for i in bidx], nb)
                sharp = upload(pool, [(m, os.path.join(sdir, _name(first + 4 * m) + ".png")) for m in sidx], 2 * nb - 1)
                clips.append(DeviceClip(folder, blurry, sharp, first, im_list))
        return cls(clips, lq_size=lq_size, rng=rng)
