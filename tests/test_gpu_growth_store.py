"""Where the fp16 x-stacked growth conv (conv_igemm_kernel<32, 3, P8, SX>) writes.  Its epilogue stages each
warpgroup's 4 output rows in shared memory and writes them with one TMA tensor store, so the tensor map's clipping is
all that keeps the right edge, the last tile row, the batch / row sub-range and the store_planes limit.  Each case
fills every plane the call neither reads nor writes with NaN and every element of its output planes with a sentinel,
then checks that the written elements match an fp64 conv within the bar below, that every other element keeps its
bits, and that a launch over many more tiles than SMs (each CTA reusing its staging buffers) gives the same bits.

Bar per element: 2^-11 |ref| (rounding to fp16) + 2^-16 sum |x w| (fp32 accumulation over <= 384 terms) + 2^-25."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
SENTINEL = -1234.0

# name: (B, H, W, sub = (b_begin, b_count, y_begin, y_count), growth planes, g_plane0, layer c, store_planes)
CASES = {
    "rows_from_5_count_19": (2, 37, 45, (0, 0, 5, 19), 16, 0, 3, 0),
    "rows_from_9_count_2": (2, 24, 64, (0, 0, 9, 2), 16, 0, 1, 0),
    "batch_from_1": (4, 20, 33, (1, 2, 0, 0), 16, 0, 2, 0),
    "batch_and_rows": (3, 29, 70, (2, 1, 3, 13), 16, 0, 0, 0),
    "store_planes_1": (2, 17, 61, (0, 0, 0, 0), 16, 0, 2, 1),
    "store_planes_2": (2, 17, 61, (0, 0, 2, 11), 16, 0, 1, 2),
    "store_planes_3": (1, 10, 30, (0, 0, 0, 0), 16, 0, 3, 3),
    "width_1": (2, 11, 1, (0, 0, 3, 5), 16, 0, 1, 0),
    "width_2": (2, 9, 2, (0, 0, 0, 0), 16, 0, 2, 0),
    "width_31": (2, 13, 31, (1, 1, 0, 0), 16, 0, 3, 0),
    "width_61": (1, 21, 61, (0, 0, 4, 15), 16, 0, 1, 0),
    "training_planes": (2, 19, 47, (0, 0, 0, 0), 16 * 12, 16 * 5, 2, 0),    # RDB 5 of a D = 12 training growth tensor
    "training_planes_sub": (3, 23, 35, (1, 2, 6, 9), 16 * 12, 16 * 11, 3, 2),
    "many_tiles": (3, 130, 72, (0, 0, 0, 0), 16, 0, 2, 0),                # ~12 tiles per SM
}


def _nchw(t):
    B, P, H, W, _ = t.shape
    return t.permute(0, 1, 4, 2, 3).reshape(B, 8 * P, H, W)


def _case(name):
    from bin_b200 import ops
    B, H, W, sub, gplanes, gp0, c, sp = CASES[name]
    gen = torch.Generator(device=DEV).manual_seed(sum(map(ord, name)))
    rnd = lambda *sh: torch.randn(*sh, device=DEV, generator=gen)
    cin = 96 + 32 * c
    x = rnd(B, 12, H, W, 8).half()
    g = torch.full((B, gplanes, H, W, 8), NAN, device=DEV).half()
    g[:, gp0:gp0 + 4 * c] = rnd(B, 4 * c, H, W, 8).half()
    op0, nstore = gp0 + 4 * c, sp if sp else 4
    g[:, op0:op0 + nstore] = SENTINEL
    w, b = rnd(32, cin, 3, 3) / (9 * cin) ** 0.5, rnd(32) * 0.1
    wp, bp = ops.pack_conv_weight(w, 32, cin), ops.pad_bias(b, 32)
    g_before = g.clone()
    ops.conv_fwd(x, wp, bp, 3, 32, in0_planes=12, in1=g, in1_plane0=gp0, in1_planes=4 * c, relu=True, out=g,
                 out_plane0=op0, sub=None if sub == (0, 0, 0, 0) else sub, store_planes=sp)
    torch.cuda.synchronize()
    # fp64 reference of the whole image, from the fp16 operands the kernel reads
    xin = torch.cat([_nchw(x), _nchw(g_before[:, gp0:gp0 + 4 * c])], 1).double()
    wd = w.half().double()
    ref = torch.relu(torch.nn.functional.conv2d(xin, wd, b.double(), padding=1))
    mag = torch.nn.functional.conv2d(xin.abs(), wd.abs(), b.double().abs(), padding=1)
    return x, g, g_before, ref, mag, (B, H, W, sub, op0, nstore)


@pytest.mark.parametrize("name", list(CASES))
def test_growth_conv_store_range(name):
    x, g, g_before, ref, mag, (B, H, W, sub, op0, nstore) = _case(name)
    b0, nb, y0, ny = sub
    nb, ny = nb or B - b0, ny or H - y0
    written = torch.zeros(g.shape[:4], dtype=torch.bool, device=DEV)            # (B, planes, H, W)
    written[b0:b0 + nb, op0:op0 + nstore, y0:y0 + ny] = True
    # every element outside the written block keeps its bits (NaN planes, input planes, sentinels)
    keep = ~written[..., None].expand_as(g)
    assert torch.equal(g.view(torch.int16)[keep], g_before.view(torch.int16)[keep])
    # the written block matches the fp64 conv
    out = _nchw(g[b0:b0 + nb, op0:op0 + nstore, y0:y0 + ny]).double()
    r = ref[b0:b0 + nb, : 8 * nstore, y0:y0 + ny]
    m = mag[b0:b0 + nb, : 8 * nstore, y0:y0 + ny]
    assert torch.isfinite(out).all() and (out >= 0).all()
    bar = 2.0 ** -11 * r.abs() + 2.0 ** -16 * m + 2.0 ** -25
    worst = ((out - r).abs() / bar).max().item()
    assert worst <= 1.0, f"{name}: worst error / bar = {worst:.3f}"


def test_growth_conv_store_same_bits_over_subranges():
    """A row band and a batch slice written by their own launches hold the bits the whole-tensor launch writes."""
    from bin_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(11)
    rnd = lambda *sh: torch.randn(*sh, device=DEV, generator=gen)
    B, H, W = 3, 45, 95
    x = rnd(B, 12, H, W, 8).half()
    g = rnd(B, 16, H, W, 8).half()
    w = rnd(32, 160, 3, 3) / (9 * 160) ** 0.5
    wp, bp = ops.pack_conv_weight(w, 32, 160), ops.pad_bias(rnd(32) * 0.1, 32)
    full, part = g.clone(), g.clone()
    run = lambda out, sub: ops.conv_fwd(x, wp, bp, 3, 32, in0_planes=12, in1=g, in1_planes=8, relu=True, out=out,
                                        out_plane0=8, sub=sub)
    run(full, None)
    for sub in ((0, 0, 0, 13), (0, 0, 13, 19), (0, 1, 32, 13), (1, 2, 32, 13)):
        run(part, sub)
    torch.cuda.synchronize()
    assert torch.equal(full.view(torch.int16), part.view(torch.int16))
