"""PNG output of the caller loop on the GPU: test.py and demo.py write every output frame with cv2.imwrite.

``encode_png`` runs one sm_90a launch sequence (bin_png_encode_u8) over up to BIN_PNG_MAX_BATCH same-size uint8
(h, w, 3) BGR images and returns complete PNG files.  Their inflated payload is the one cv2.imwrite writes (every row
filtered with Sub, deflate with zlib's Z_RLE parse), so any decoder returns the same pixels; the compressed size stays
close to cv2's.  The bytes depend only on the pixels and (h, w).

  * ``encode_png_async`` returns a handle at once; its ``result()`` waits only for that encode's copy to pinned host
    memory, so a loop can write window k's files while window k+1 runs on the GPU.
  * ``imwrite`` is cv2.imwrite for a .png path with default params and a uint8 (h, w, 3) numpy array or CUDA tensor.
  * ``install_cv2_imwrite()`` routes those calls of cv2.imwrite here and every other call to the original function.
Anything else raises BinB200Error: there is no CPU encoder in the package."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from ._lib import BIN_PNG_MAX_BATCH, BinB200Error, check, lib


def _check_batch(imgs, fn: str):
    if isinstance(imgs, torch.Tensor):
        imgs = [imgs]
    imgs = list(imgs)
    if not imgs:
        raise BinB200Error(f"{fn}: no images given")
    for x in imgs:
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise BinB200Error(f"{fn}: CUDA tensors only (bin_b200 has no CPU path)")
        if x.dtype != torch.uint8:
            raise BinB200Error(f"{fn}: uint8 images only, got {x.dtype}")
        if x.dim() != 3 or x.shape[2] != 3:
            raise BinB200Error(f"{fn}: images must be (h, w, 3) BGR, got {tuple(x.shape)}")
        if not x.is_contiguous():
            raise BinB200Error(f"{fn}: images must be contiguous (row pitch 3w)")
    shape, dev = tuple(imgs[0].shape), imgs[0].device
    for x in imgs[1:]:
        if tuple(x.shape) != shape:
            raise BinB200Error(f"{fn}: all images of one call must have the same size, got {shape} and {tuple(x.shape)}")
        if x.device != dev:
            raise BinB200Error(f"{fn}: images on different devices ({dev}, {x.device})")
    h, w = shape[0], shape[1]
    if int(lib().bin_png_max_bytes(h, w)) == 0:
        raise BinB200Error(f"{fn}: size {h}x{w} is out of range (1 <= h, w <= 65535, h*(3w+1) < 2^31)")
    return imgs, h, w, dev


class PngBatch:
    """An encode in flight.  It holds the device output, the workspace and the pinned copy until ``result()``, so none
    of them is reused before the copy completes."""

    def __init__(self, parts):
        self._parts = parts             # [(event, pinned files, pinned sizes, stride, n, device buffers)]
        self._files = None

    def done(self) -> bool:
        return all(ev.query() for ev, *_ in self._parts)

    def result(self) -> list:
        """-> list of bytes, one PNG file per image, in the order given."""
        if self._files is None:
            files = []
            for ev, host, sizes, stride, n, _ in self._parts:
                ev.synchronize()
                buf = host.numpy()
                for i, size in enumerate(sizes.tolist()[:n]):
                    files.append(buf[i * stride:i * stride + size].tobytes())
            self._files, self._parts = files, []
        return self._files


def encode_png_async(imgs) -> PngBatch:
    """imgs: a list of device uint8 (h, w, 3) BGR tensors of one size (or one tensor), contiguous, on one device.
    Enqueues the encode and the copy to pinned host memory on the current stream, one launch sequence per
    BIN_PNG_MAX_BATCH images, and returns a handle whose ``result()`` gives the files."""
    imgs, h, w, dev = _check_batch(imgs, "encode_png")
    L = lib()
    stride = (int(L.bin_png_max_bytes(h, w)) + 255) // 256 * 256
    parts = []
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream()
        for k in range(0, len(imgs), BIN_PNG_MAX_BATCH):
            group = imgs[k:k + BIN_PNG_MAX_BATCH]
            n = len(group)
            out = torch.empty(n * stride, dtype=torch.uint8, device=dev)
            sizes = torch.empty(n, dtype=torch.int64, device=dev)
            ws = torch.empty(max(int(L.bin_png_workspace_bytes(n, h, w)), 1), dtype=torch.uint8, device=dev)
            ptrs = (C.c_void_p * n)(*[x.data_ptr() for x in group])
            check(L.bin_png_encode_u8(ptrs, n, h, w, out.data_ptr(), stride, sizes.data_ptr(), ws.data_ptr(), ws.numel(),
                                      stream.cuda_stream))
            host = torch.empty(n * stride, dtype=torch.uint8, pin_memory=True)
            host_sizes = torch.empty(n, dtype=torch.int64, pin_memory=True)
            host.copy_(out, non_blocking=True)
            host_sizes.copy_(sizes, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(stream)
            parts.append((ev, host, host_sizes, stride, n, (out, sizes, ws, group)))
    return PngBatch(parts)


def encode_png(imgs) -> list:
    """encode_png_async(imgs).result(): a list of bytes, one PNG file per image."""
    return encode_png_async(imgs).result()


# ----------------------------------------------------------------------------- cv2.imwrite
def _is_png_path(path) -> bool:
    return isinstance(path, (str, os.PathLike)) and os.fspath(path).lower().endswith(".png")


def _covered(img) -> bool:
    if isinstance(img, torch.Tensor):
        return img.is_cuda and img.dtype == torch.uint8 and img.dim() == 3 and img.shape[2] == 3
    return isinstance(img, np.ndarray) and img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3


def imwrite(path, img, params=None) -> bool:
    """cv2.imwrite for a .png path with default params: img is a uint8 (h, w, 3) BGR numpy array (uploaded to the
    current device) or CUDA tensor.  -> True once the file is written, False when it cannot be opened (as cv2)."""
    if not _is_png_path(path):
        raise BinB200Error(f"imwrite: only .png paths are supported, got {path!r}")
    if params is not None and len(params) > 0:
        raise BinB200Error(f"imwrite: params={params!r} are not supported (only the defaults)")
    if not _covered(img):
        raise BinB200Error("imwrite: a uint8 (h, w, 3) numpy array or CUDA tensor is required")
    if isinstance(img, np.ndarray):
        if not torch.cuda.is_available():
            raise BinB200Error("imwrite: no CUDA device (bin_b200 has no CPU path)")
        img = torch.from_numpy(np.ascontiguousarray(img)).to(torch.cuda.current_device())
    data = encode_png([img])[0]
    try:
        with open(os.fspath(path), "wb") as fh:
            fh.write(data)
    except OSError:
        return False
    return True


def install_cv2_imwrite():
    """Replace cv2.imwrite with a wrapper that sends .png writes of uint8 (h, w, 3) images with default params to
    ``imwrite`` above and every other call (another extension, params, other dtypes or shapes) to the original
    function unchanged.  Idempotent.  -> the cv2 module."""
    import cv2
    if getattr(cv2.imwrite, "_bin_b200_original", None) is not None:
        return cv2
    original = cv2.imwrite

    def imwrite_wrapper(*args, **kwargs):
        a = dict(zip(("filename", "img", "params"), args))
        if len(args) <= 3 and not (set(kwargs) - {"filename", "img", "params"}) and not (set(a) & set(kwargs)):
            a.update(kwargs)
            path, img, params = a.get("filename"), a.get("img"), a.get("params")
            if _is_png_path(path) and (params is None or len(params) == 0) and _covered(img) \
                    and int(lib().bin_png_max_bytes(img.shape[0], img.shape[1])) > 0:
                return imwrite(path, img)
        return original(*args, **kwargs)

    imwrite_wrapper._bin_b200_original = original
    imwrite_wrapper.__doc__ = "cv2.imwrite; .png writes of uint8 (h, w, 3) images with default params run on the GPU"
    cv2.imwrite = imwrite_wrapper
    return cv2
