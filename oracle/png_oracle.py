"""Test-only restatement of what cv2.imwrite writes for a uint8 (h, w, 3) image at a .png path (cv2 4.x on libpng and
zlib, default params), and a strict PNG reader built on the standard library alone.

  * IHDR (w, h, bit depth 8, colour type 2, compression 0, filter 0, interlace 0), IDAT chunks of 8192 data bytes (the
    last one shorter), IEND; no other chunk.
  * The file stores RGB (libpng swaps cv2's BGR on write).  Every row uses filter type 1 (Sub): the byte 1, then the
    row's RGB bytes minus the byte 3 positions to the left, mod 256 (the first pixel as is).  Rows of one pixel use
    filter type 0 (libpng drops Sub when the width is 1; the filtered bytes are the same).
  * The zlib stream is deflate at level 1, strategy Z_RLE, memLevel 8.  From 64x128 up it is byte-identical to
    zlib.compressobj(1, DEFLATED, 15, 8, Z_RLE) over that payload; below, libpng shrinks the window (other header
    bytes, same payload)."""
from __future__ import annotations

import struct
import zlib

import numpy as np

SIGNATURE = b"\x89PNG\r\n\x1a\n"
IDAT_BYTES = 8192


def payload(img) -> bytes:
    """The inflated IDAT payload cv2.imwrite writes for a uint8 (h, w, 3) BGR image: the file stores RGB, and rows of
    one pixel use filter type 0 (libpng drops Sub there; the bytes are the same)."""
    a = np.ascontiguousarray(img, dtype=np.uint8)
    h, w, c = a.shape
    assert c == 3
    rows = np.ascontiguousarray(a[:, :, ::-1]).reshape(h, 3 * w)
    sub = rows.copy()
    sub[:, 3:] = rows[:, 3:] - rows[:, :-3]               # uint8 arithmetic wraps mod 256
    return np.concatenate([np.full((h, 1), 0 if w == 1 else 1, np.uint8), sub], axis=1).tobytes()


def file_bytes(zlen: int) -> int:
    """Size of a file whose zlib stream has zlen bytes: signature, IHDR, the IDAT chunks, IEND."""
    return 8 + 25 + 12 * ((zlen + IDAT_BYTES - 1) // IDAT_BYTES) + zlen + 12


def cv2_like_size(img) -> int:
    """File size cv2.imwrite gives (exact from 64x128 up, on the zlib version cv2 was recorded with)."""
    co = zlib.compressobj(1, zlib.DEFLATED, 15, 8, zlib.Z_RLE)
    z = co.compress(payload(img)) + co.flush()
    return file_bytes(len(z))


def stored_size(h: int, w: int, segment: int) -> int:
    """File size when the payload goes out as stored deflate blocks of `segment` bytes (5 bytes of block header each)."""
    n = h * (3 * w + 1)
    nseg = -(-n // segment)
    return file_bytes(2 + 5 * nseg + n + 4)


def parse_png(data: bytes):
    """Strict reader of an 8-bit truecolour, non-interlaced PNG: checks the signature, the IHDR fields, every CRC, the
    chunk order (IHDR, one or more consecutive IDAT, IEND, nothing else and nothing after), the zlib header, the
    Adler-32 and that no data trails the stream, and that every row's filter is Sub (None for one-pixel rows).
    -> (payload bytes, uint8 (h, w, 3) pixels in BGR order, as cv2.imread returns them).  Raises ValueError on any
    violation."""
    data = bytes(data)
    if data[:8] != SIGNATURE:
        raise ValueError("bad signature")
    pos, chunks = 8, []
    while pos < len(data):
        if pos + 12 > len(data):
            raise ValueError("truncated chunk")
        (n,) = struct.unpack(">I", data[pos:pos + 4])
        kind, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        if len(body) != n or pos + 12 + n > len(data):
            raise ValueError("truncated chunk")
        (crc,) = struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])
        if zlib.crc32(kind + body) != crc:
            raise ValueError(f"bad CRC in {kind!r}")
        chunks.append((kind, body))
        pos += 12 + n
        if kind == b"IEND":
            break
    if pos != len(data):
        raise ValueError("data after IEND")
    kinds = [k for k, _ in chunks]
    if len(kinds) < 3 or kinds[0] != b"IHDR" or kinds[-1] != b"IEND" or any(k != b"IDAT" for k in kinds[1:-1]):
        raise ValueError(f"bad chunk order {kinds}")
    ihdr = chunks[0][1]
    if len(ihdr) != 13:
        raise ValueError("bad IHDR length")
    w, h, depth, ctype, comp, filt, interlace = struct.unpack(">IIBBBBB", ihdr)
    if not (w > 0 and h > 0 and depth == 8 and ctype == 2 and comp == 0 and filt == 0 and interlace == 0):
        raise ValueError(f"unsupported IHDR {(w, h, depth, ctype, comp, filt, interlace)}")
    if chunks[-1][1]:
        raise ValueError("IEND with data")
    z = b"".join(b for _, b in chunks[1:-1])
    if len(z) < 6 or z[0] & 0x0F != 8 or z[0] >> 4 > 7 or ((z[0] << 8) | z[1]) % 31 or z[1] & 0x20:
        raise ValueError("bad zlib header")
    d = zlib.decompressobj(-15)
    raw = d.decompress(z[2:])
    if not d.eof:
        raise ValueError("truncated deflate stream")
    tail = d.unused_data
    if len(tail) != 4:
        raise ValueError(f"{len(tail)} bytes after the deflate stream (want the 4-byte Adler-32)")
    if struct.unpack(">I", tail)[0] != zlib.adler32(raw):
        raise ValueError("bad Adler-32")
    rowlen = 3 * w + 1
    if len(raw) != h * rowlen:
        raise ValueError(f"payload of {len(raw)} bytes, want {h * rowlen}")
    rows = np.frombuffer(raw, np.uint8).reshape(h, rowlen)
    if not (rows[:, 0] == (0 if w == 1 else 1)).all():
        raise ValueError("a row does not use filter type 1 (Sub), or 0 for one-pixel rows")
    sub = rows[:, 1:].reshape(h, w, 3).astype(np.uint8)
    pix = np.cumsum(sub, axis=1, dtype=np.uint64) % 256              # undo Sub per channel
    return raw, np.ascontiguousarray(pix.astype(np.uint8)[:, :, ::-1])
