"""How the persistent fused RDB tail (rdb_tail.cu) walks its tiles: one CTA per SM, each walking tiles blockIdx.x,
+gridDim.x, ... through a 5-stage ring of 6 activation chunks per tile.  Each case is bit-identical to conv3 and the LFF
run as two launches, and leaves a sentinel in every element it must not write: the output planes outside
[out_plane0, out_plane0 + 12) and the rows outside the sub-range.  The tile counts are chosen against the grid: one
tile, a grid one short or one over, an odd and an even number of tiles per CTA, many laps of the ring, and a grid
capped at 3 CTAs with hundreds of tiles each."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 7.0
OUT_PLANES, OUT_PLANE0 = 16, 2          # the tail writes planes [2, 14) of a 16-plane tensor


def _tail_vs_layerwise(B, H, W, sub):
    """Runs the fused tail and the two-launch path on the same random operands; returns (fused, layerwise, g, g_before,
    rows) with `rows` the (B, H) mask of the rows the call may write."""
    from bin_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(B * 7919 + H * 31 + W)
    rnd = lambda *sh: torch.randn(*sh, device="cuda", generator=gen)
    x, g = rnd(B, 12, H, W, 8).half(), rnd(B, 16, H, W, 8).half()
    w3, wl = rnd(32, 192, 3, 3) / 1728 ** 0.5, rnd(96, 224, 1, 1) / 224 ** 0.5
    b3, bl = ops.pad_bias(rnd(32) * 0.1, 32), ops.pad_bias(rnd(96) * 0.1, 96)
    p3, pl = ops.pack_conv_weight(w3, 32, 192), ops.pack_conv_weight(wl, 96, 224)
    g_before, g_ref = g.clone(), g.clone()
    out = torch.full((B, OUT_PLANES, H, W, 8), SENTINEL, device="cuda").half()
    out_ref = out.clone()
    s4 = None if sub == (0, 0, 0, 0) else sub
    ops.conv_fwd(x, p3, b3, 3, 32, in0_planes=12, in1=g_ref, in1_planes=12, relu=True, out=g_ref, out_plane0=12, sub=s4)
    ops.conv_fwd(x, pl, bl, 1, 96, in0_planes=12, in1=g_ref, in1_planes=16, out=out_ref, out_plane0=OUT_PLANE0, res=x,
                 sub=s4)
    ops.rdb_tail_fwd(x, g, p3, b3, pl, bl, out, out_plane0=OUT_PLANE0, sub=sub)
    torch.cuda.synchronize()
    b0, nb, y0, ny = sub
    rows = torch.zeros(B, H, dtype=torch.bool)
    rows[b0:(b0 + nb) if nb else B, y0:(y0 + ny) if ny else H] = True
    return out, out_ref, g, g_before, rows


def _check(B, H, W, sub=(0, 0, 0, 0)):
    out, out_ref, g, g_before, rows = _tail_vs_layerwise(B, H, W, sub)
    assert torch.equal(g, g_before)                                   # inputs untouched, g3 never written
    assert torch.equal(out, out_ref)
    outside = torch.ones(OUT_PLANES, dtype=torch.bool)
    outside[OUT_PLANE0:OUT_PLANE0 + 12] = False
    assert (out[:, outside] == SENTINEL).all()
    written = (out != SENTINEL).any(dim=(1, 3, 4)).cpu()
    assert not (written & ~rows).any()
    assert written[rows].float().mean() > 0.99                        # random outputs: every row in range is written


def _grid():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("B,H,W,sub", [(1, 4, 30, (0, 0, 0, 0)),           # one full tile
                                       (1, 3, 17, (0, 0, 0, 0)),           # one ragged tile
                                       (2, 9, 40, (1, 1, 5, 1))])          # one tile inside a batch / row sub-range
def test_single_tile(B, H, W, sub):
    _check(B, H, W, sub)


@pytest.mark.parametrize("ntiles", ["grid-1", "grid+1", "2grid+1"])
def test_tiles_around_the_grid(ntiles):
    """30-column tensors have one tile column, so H = 4 n gives exactly n tiles: the grid is then min(n, SMs)."""
    n = {"grid-1": _grid() - 1, "grid+1": _grid() + 1, "2grid+1": 2 * _grid() + 1}[ntiles]
    _check(1, 4 * n - 1, 30)                                          # last tile row ragged


@pytest.mark.parametrize("per_cta", [3, 4])
def test_odd_and_even_tiles_per_cta(per_cta):
    """Every CTA runs `per_cta` tiles, so each CTA ends its walk at a different ring slot and mbarrier phase."""
    _check(per_cta, 4 * _grid(), 30)


def test_ring_wraps_many_times():
    """2 x 100 x 8 = 1600 tiles, 12-13 per CTA: about 75 chunks through the 5-stage ring, on ragged tiles in x."""
    _check(2, 400, 227)
    _check(3, 150, 233, (1, 2, 17, 121))


def _child(code, env):
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % ROOT + code],
                       env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout


def test_three_sms_hundreds_of_tiles_per_cta():
    """BIN_B200_MAX_SMS=3 caps every grid at 3 CTAs: 2 x 33 x 9 = 594 tiles, 198 per CTA (the library reads the switch
    once per process, hence a child)."""
    code = ("import importlib.util\n"
            "spec = importlib.util.spec_from_file_location('rdb_tail_tiles', %r)\n"
            "mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod); _check = mod._check\n" % __file__ +
            "_check(2, 130, 250)\n"
            "_check(2, 130, 250, (1, 1, 3, 101))\n"
            "print('OK')\n")
    assert _child(code, {"BIN_B200_MAX_SMS": "3"}).strip().endswith("OK")

