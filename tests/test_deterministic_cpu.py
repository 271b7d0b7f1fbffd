"""BIN_DETERMINISTIC without a device: the flag checks and scratch-size queries of the *_ex entry points, the gradient
workspace that holds the bias-gradient partials, and the BIN_B200_MAX_SMS floor of the wgrad workspace.  Every call
here is invalid and must fail before anything reaches a device: a call that got as far as a launch would fail with
BIN_ERR_CUDA."""
import ctypes as C
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DET = 1
SLAB = 128 * 512 * 4                      # one wgrad CTA's accumulator slab, bytes


@pytest.fixture(scope="module")
def L():
    from bin_b200 import _lib
    assert _lib.BIN_DETERMINISTIC == DET
    return _lib.lib()


def _err(L, rc):
    return rc, L.bin_last_error().decode()


def _ptrs(n, p):
    return (C.c_void_p * n)(*([p] * n))


def test_pixel_loss_scratch_size(L):
    for npairs, n in ((17, 1), (17, 4096), (17, 4097), (17, 256 * 4096), (17, 256 * 4096 * 2 + 3), (1, 10 ** 9)):
        blocks = min((n + 4095) // 4096, 256)
        assert L.bin_pixel_loss_scratch_bytes(npairs, n) == npairs * blocks * 4
    assert L.bin_pixel_loss_scratch_bytes(0, 100) == 0 and L.bin_pixel_loss_scratch_bytes(21, 100) == 0


def test_pixel_loss_ex_checks(L):
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    a, b = _ptrs(17, p), _ptrs(17, p)
    n = 256 * 4096 * 2 + 3
    need = L.bin_pixel_loss_scratch_bytes(17, n)

    def call(flags, scratch, nbytes):
        return _err(L, L.bin_pixel_loss_fwd_ex(a, b, 17, n, 2, 1e-6, p, flags, scratch, nbytes, None))

    assert call(DET, None, need) == (1, "pixel_loss: BIN_DETERMINISTIC needs a scratch buffer")
    assert call(DET, p, need - 1) == (4, "pixel_loss: scratch too small")
    assert call(2, p, need) == (1, "pixel_loss_fwd: unknown flags")
    assert call(DET | 4, p, need) == (1, "pixel_loss_fwd: unknown flags")
    rc = L.bin_pixel_loss_fwd_ex(a, b, 21, n, 2, 1e-6, p, DET, p, need, None)
    assert _err(L, rc) == (1, "pixel_loss: bad pair count / kind")


def test_convlstm_scratch_size(L):
    for B, H, W in ((1, 1, 1), (2, 12, 14), (2, 96, 128), (8, 256, 256)):
        blocks = min((B * H * W + 31) // 32, 592)
        assert L.bin_convlstm_bwd_scratch_bytes(B, H, W) == blocks * 660 * 4
    assert L.bin_convlstm_bwd_scratch_bytes(8, 256, 256) <= 592 * 660 * 4
    assert L.bin_convlstm_bwd_scratch_bytes(0, 4, 4) == 0


def test_convlstm_bwd_ex_checks(L):
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    B, H, W = 2, 96, 128
    need = L.bin_convlstm_bwd_scratch_bytes(B, H, W)

    def call(flags, scratch, nbytes):
        return _err(L, L.bin_convlstm_bwd_ex(p, p, p, p, p, p, p, p, p, p, p, p, p, B, H, W, flags, scratch, nbytes, None))

    assert call(DET, None, need) == (1, "convlstm_bwd: BIN_DETERMINISTIC needs a scratch buffer")
    assert call(DET, p, need - 4) == (4, "convlstm_bwd: scratch too small")
    assert call(8, p, need) == (1, "convlstm_bwd: unknown flags")


def _frames(ncalls, nframes, Bc):
    from bin_b200 import _lib
    f = _lib.Frames()
    f.ncalls, f.nframes, f.Bc = ncalls, nframes, Bc
    return f


def test_backbone_bwd_ex_rejects_unknown_flags(L):
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    n, ncalls, Bc, H, W = 3, 2, 1, 32, 48
    dout, dfr = _frames(ncalls, n, Bc), _frames(ncalls, n, Bc)
    gws = L.bin_backbone_grad_workspace_bytes(n, ncalls * Bc, H, W)
    rc = L.bin_backbone_bwd_ex(n, p, C.byref(dout), C.byref(dfr), H, W, p, p, gws, p, p, 2, None)
    assert _err(L, rc) == (1, "backbone_bwd: unknown flags")
    fwd = L.bin_backbone_workspace_bytes(n, ncalls * Bc, H, W)
    aligned = (p + 255) // 256 * 256 + 4096
    rc = L.bin_backbone_bwd_recompute_ex(n, p, p, C.byref(dout), C.byref(dfr), H, W, aligned, fwd, p, gws, p, p, 6, None)
    assert _err(L, rc) == (1, "backbone_bwd: unknown flags")
    rc = L.bin_backbone_bwd_ex(n, None, C.byref(dout), C.byref(dfr), H, W, p, p, gws, p, p, DET, None)
    assert _err(L, rc) == (1, "backbone_bwd: null argument")


def _grad_ws_without_partials(n, Btot, H, W):
    """Bytes of the gradient workspace's activation-gradient regions (api.cu grad_ws), each 256-byte aligned."""
    up = lambda v: (v + 255) // 256 * 256
    h, w = H // 2, W // 2
    x0 = ((12 * n + 31) // 32 * 32) // 8
    regions = [(4, H, W), (8, H, W), (32, h, w), (12, h, w), (12, h, w), (144, h, w), (12, h, w), (16, h, w), (x0, h, w)]
    off = 0
    for planes, hh, ww in regions:
        off = up(off + Btot * planes * hh * ww * 16)
    return off


def test_grad_workspace_holds_the_bias_partials(L):
    """The deterministic bias-gradient partials ([B][blocks of 1024 px][C], largest for UPNet.0's 256 channels at low
    resolution or UPNet.2's 3 at full resolution) share the wgrad slabs; the region grows when they would not fit."""
    slabs = 132 * SLAB
    for n, Btot, H, W in ((3, 12, 256, 256), (5, 8, 352, 640), (2, 36, 2048, 4096), (3, 6, 4096, 4096)):
        bias = 4 * max(Btot * ((H * W + 1023) // 1024) * 3, Btot * ((H // 2 * (W // 2) + 1023) // 1024) * 256)
        region = (max(slabs, bias) + 255) // 256 * 256
        assert L.bin_backbone_grad_workspace_bytes(n, Btot, H, W) == _grad_ws_without_partials(n, Btot, H, W) + region
    assert L.bin_conv_wgrad_workspace_bytes() == slabs


def test_max_sms_keeps_the_deterministic_slabs():
    """BIN_B200_MAX_SMS lowers the grids the library sizes by SM count, but the wgrad workspace always holds the 132
    slabs of the deterministic grid."""
    code = ("import sys; sys.path.insert(0, %r)\n"
            "from bin_b200 import _lib\n"
            "print('BYTES', _lib.lib().bin_conv_wgrad_workspace_bytes())\n" % ROOT)
    for cap in ("66", "1"):
        env = dict(os.environ, BIN_B200_MAX_SMS=cap)
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        assert int(r.stdout.split("BYTES")[-1]) == 132 * SLAB
