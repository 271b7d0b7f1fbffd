"""Generate tests/golden/png.npz with cv2.imencode('.png') (cv2.imwrite's encoder) on seeded images.

Run where cv2 is importable:

    python oracle/make_golden_png.py

The fixture stores each image, the file cv2 wrote for it, the cv2 version, the zlib version cv2 reports and the zlib
runtime version of the Python that made it (the stdlib-zlib restatement in png_oracle.cv2_like_size is only compared
byte for byte on that version)."""
import os
import re
import zlib

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "png.npz")


def from_sub(sub):
    """The BGR image whose Sub-filtered rows (RGB, as the file stores them) are `sub` ((h, 3w) bytes): a running sum
    per channel, mod 256."""
    h, n = sub.shape
    rgb = (np.cumsum(sub.reshape(h, n // 3, 3).astype(np.uint64), axis=1) % 256).astype(np.uint8)
    return np.ascontiguousarray(rgb[:, :, ::-1])


def smooth(rng, h, w):
    from scipy.ndimage import gaussian_filter
    z = gaussian_filter(rng.standard_normal((h, w, 3)), sigma=(4.0, 4.0, 0.0))
    z = (z - z.min()) / (z.max() - z.min())
    return np.clip(np.round(z * 235 + 10), 0, 255).astype(np.uint8)


def images(rng):
    yield "noise_96x160", rng.integers(0, 256, size=(96, 160, 3), dtype=np.uint8)
    yield "flat_64x128", np.full((64, 128, 3), (30, 120, 200), np.uint8)
    yield "smooth_96x160", smooth(rng, 96, 160)
    x = np.arange(128)
    yield "stripes_64x128", np.repeat(np.where((x // 5) % 2, 220, 17).astype(np.uint8)[None, :, None], 64, 0).repeat(3, 2)
    # Sub bytes: a non-zero byte, then r + 1 zeros (a run of r bytes that repeat the previous one), r = 257..261
    sub = rng.integers(1, 256, size=(96, 480), dtype=np.uint8)
    for y in range(96):
        r = 257 + y % 5
        start = int(rng.integers(1, 480 - r - 1))
        sub[y, start:start + r + 1] = 0
    yield "runs_96x160", from_sub(sub)
    yield "ones_64x128", from_sub(np.ones((64, 384), np.uint8))       # the whole payload is the byte 1: one run
    yield "px_1x1", np.array([[[7, 250, 128]]], np.uint8)
    yield "small_7x9", rng.integers(0, 256, size=(7, 9, 3), dtype=np.uint8)


def main():
    rng = np.random.default_rng(2026)
    rec, names = {}, []
    for name, img in images(rng):
        ok, buf = cv2.imencode(".png", img)
        assert ok
        rec[f"{name}_img"] = img
        rec[f"{name}_png"] = np.frombuffer(buf.tobytes(), np.uint8)
        names.append(name)
        print(f"{name:16s} {img.shape} -> {buf.size} bytes")
    info = cv2.getBuildInformation()
    m = re.search(r"ZLib:\s*(.*)", info)
    rec["names"] = np.array(names)
    rec["cv2_version"] = np.array(cv2.__version__)
    rec["cv2_zlib"] = np.array(m.group(1).strip() if m else "unknown")
    rec["zlib_runtime_version"] = np.array(zlib.ZLIB_RUNTIME_VERSION)
    np.savez_compressed(OUT, **rec)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", rec["cv2_zlib"], "/ python zlib", zlib.ZLIB_RUNTIME_VERSION)


if __name__ == "__main__":
    main()
