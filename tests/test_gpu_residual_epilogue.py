"""P8 convs with a residual, run in place: `out` and `res` the same tensor and the same planes.

The fp16 epilogue loads each accumulator row set's residual one row set ahead: row set (0, 0) during the tile's last K
stage, row set k + 1 before the stores of row set k.  That is exact in place because row sets are disjoint pixels and
each thread reads and writes only its own fragment's pixels.  Here the in-place result must equal the out-of-place one
bit for bit, and the planes the call does not write must keep theirs.  The shape's last tile row and tile column are
partial (H = 13 against 8-row tiles, W = 47 against 30- and 32-pixel tiles), with more than one image.
"""
import pytest
import torch

from bin_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
B, H, W = 2, 13, 47
PLANE0 = 4                     # the written planes start inside the tensor, so planes on both sides must keep their bits


@pytest.mark.parametrize("x3", [False, True], ids=["fp16", "x3"])
@pytest.mark.parametrize("cout,k", [(96, 3), (96, 1), (64, 3)], ids=["96x3", "96x1", "64x3"])
def test_in_place_residual_matches_out_of_place(cout, k, x3):
    g = torch.Generator(device="cpu").manual_seed(cout * 10 + k)
    f = 2 if x3 else 1
    cin = 96
    n = cout // 8
    w = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(DEV)
    bias = ops.pad_bias((torch.randn(cout, generator=g) * 0.1).to(DEV), cout)
    wp = ops.pack_conv_weight(w, cout, cin, 0, prec=1 if x3 else 0)
    x = (torch.randn(B, f * cin // 8, H, W, 8, generator=g) * 0.5).half().to(DEV)
    res0 = (torch.randn(B, f * (PLANE0 + n + 4), H, W, 8, generator=g) * 0.5).half().to(DEV)

    out = res0.clone()                  # out of place: the residual is read from res0, the result written here
    ops.conv_fwd(x, wp, bias, k, cout, out=out, out_plane0=PLANE0, res=res0, res_plane0=PLANE0, x3=x3)
    inplace = res0.clone()
    ops.conv_fwd(x, wp, bias, k, cout, out=inplace, out_plane0=PLANE0, res=inplace, res_plane0=PLANE0, x3=x3)
    torch.cuda.synchronize()

    assert not torch.equal(out, res0)   # the call wrote something
    assert torch.equal(inplace.view(torch.int16), out.view(torch.int16))
