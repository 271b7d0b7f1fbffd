"""PNG output without a device: the oracle against the cv2 fixture, the strict reader's refusals, the worst-case size
query and the argument checks of bin_png_encode_u8 (all of which come before its first CUDA call)."""
import ctypes as C
import os
import struct
import zlib

import numpy as np
import pytest

from oracle import png_oracle as P

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "png.npz")
ERR_ARG, ERR_WORKSPACE = 1, 4


@pytest.fixture(scope="module")
def G():
    return np.load(GOLDEN)


def _cases(G):
    return [(str(n), G[f"{n}_img"], G[f"{n}_png"].tobytes()) for n in G["names"]]


def test_oracle_payload_is_cv2s(G):
    for name, img, png in _cases(G):
        raw, pix = P.parse_png(png)
        assert raw == P.payload(img), name
        assert np.array_equal(pix, img), name


def test_size_restatement_matches_cv2(G):
    if zlib.ZLIB_RUNTIME_VERSION != str(G["zlib_runtime_version"]):
        pytest.skip(f"fixture made with zlib {G['zlib_runtime_version']}, running {zlib.ZLIB_RUNTIME_VERSION}")
    n = 0
    for name, img, png in _cases(G):
        if img.shape[0] >= 64 and img.shape[1] >= 128:
            assert P.cv2_like_size(img) == len(png), name
            n += 1
    assert n >= 5


def _chunks(data):
    pos, out = 8, []
    while pos < len(data):
        (n,) = struct.unpack(">I", data[pos:pos + 4])
        out.append((pos, data[pos + 4:pos + 8], n))
        pos += 12 + n
    return out


def _rebuild(img, z):
    """A well-formed file around the zlib stream z (valid CRCs), for testing the reader's zlib checks."""
    h, w = img.shape[:2]

    def chunk(kind, body):
        return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body))
    out = P.SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0))
    for k in range(0, len(z), P.IDAT_BYTES):
        out += chunk(b"IDAT", z[k:k + P.IDAT_BYTES])
    return out + chunk(b"IEND", b"")


def test_parse_png_rejects_damage(G):
    _, img, png = _cases(G)[2]                      # smooth_96x160: several IDAT chunks
    pos, kind, n = _chunks(png)[1]
    assert kind == b"IDAT"
    bad = bytearray(png)
    bad[pos + 8 + n] ^= 0x01                        # a CRC byte
    with pytest.raises(ValueError, match="CRC"):
        P.parse_png(bytes(bad))
    z = zlib.compress(P.payload(img), 1)
    assert P.parse_png(_rebuild(img, z))[0] == P.payload(img)
    with pytest.raises(ValueError, match="truncated"):
        P.parse_png(_rebuild(img, z[:len(z) // 2]))
    with pytest.raises(ValueError, match="Adler"):
        P.parse_png(_rebuild(img, z[:-1] + bytes([z[-1] ^ 0x40])))
    with pytest.raises(ValueError, match="after the deflate stream"):
        P.parse_png(_rebuild(img, z + b"\0"))
    with pytest.raises(ValueError, match="signature"):
        P.parse_png(b"\0" + png[1:])
    with pytest.raises(ValueError, match="after IEND"):
        P.parse_png(png + b"\0")


@pytest.fixture(scope="module")
def L():
    from bin_b200 import _lib
    return _lib.lib()


@pytest.mark.parametrize("h,w", [(1, 1), (1, 2), (2, 1), (7, 9), (64, 128), (720, 1280), (768, 1344), (2160, 3840),
                                 (1, 65535), (10922, 65535)])
def test_max_bytes_bounds_all_stored(L, h, w):
    got = int(L.bin_png_max_bytes(h, w))
    assert got >= P.stored_size(h, w, 32768)
    assert got >= P.stored_size(h, w, 65535)        # any stored blocks no larger than deflate allows
    assert got <= P.stored_size(h, w, 32768) + 8
    assert int(L.bin_png_workspace_bytes(1, h, w)) > 0


def test_max_bytes_out_of_range(L):
    for h, w in ((0, 5), (5, 0), (-1, 5), (65536, 1), (1, 65536), (65535, 65535), (10923, 65535)):
        assert L.bin_png_max_bytes(h, w) == 0, (h, w)
        assert L.bin_png_workspace_bytes(1, h, w) == 0, (h, w)
    assert L.bin_png_workspace_bytes(0, 8, 8) == 0
    assert L.bin_png_workspace_bytes(17, 8, 8) == 0


def test_encode_argument_checks_without_device(L):
    from bin_b200._lib import BIN_PNG_MAX_BATCH
    h, w = 8, 8
    fake = 1 << 20                                   # never dereferenced: every check precedes the first CUDA call
    stride = int(L.bin_png_max_bytes(h, w))
    ws = int(L.bin_png_workspace_bytes(2, h, w))
    ptrs = (C.c_void_p * 2)(fake, fake)

    def call(ptrs=ptrs, n=2, h=h, w=w, out=fake, stride=stride, sizes=fake, ws_ptr=fake, ws_bytes=ws):
        rc = L.bin_png_encode_u8(ptrs, n, h, w, out, stride, sizes, ws_ptr, ws_bytes, None)
        return rc, L.bin_last_error().decode()

    assert call(ptrs=None)[0] == ERR_ARG
    assert call(out=None)[0] == ERR_ARG
    assert call(sizes=None)[0] == ERR_ARG
    assert call(ws_ptr=None)[0] == ERR_ARG
    assert call(ptrs=(C.c_void_p * 2)(fake, None))[0] == ERR_ARG
    assert call(n=0)[0] == ERR_ARG
    big = (C.c_void_p * (BIN_PNG_MAX_BATCH + 1))(*([fake] * (BIN_PNG_MAX_BATCH + 1)))
    assert call(ptrs=big, n=BIN_PNG_MAX_BATCH + 1)[0] == ERR_ARG
    for hh, ww in ((0, 8), (8, 0), (65536, 8), (8, 65536), (10923, 65535)):
        rc, msg = call(h=hh, w=ww)
        assert rc == ERR_ARG and "h and w" in msg, (hh, ww, msg)
    rc, msg = call(stride=stride - 1)
    assert rc == ERR_ARG and "out_stride" in msg
    rc, msg = call(stride=2 ** 63)
    assert rc == ERR_ARG and "overflows" in msg
    assert call(ws_ptr=fake + 8)[0] == ERR_ARG
    assert call(sizes=fake + 4)[0] == ERR_ARG
    rc, msg = call(ws_bytes=ws - 1)
    assert rc == ERR_WORKSPACE and "workspace" in msg
