"""The window's layers outside the RDBs at awkward shapes, against fp64, with the forward fuzz's sentinel discipline.

  pixshuf   UPNet.0 <128,3> + PixelShuffle(2): the epilogue stages each accumulator row set in shared memory and writes
            whole 16-byte full-res pixels.  W not a multiple of the 30-pixel tile, tile rows not a multiple of 8, B up to
            3, out_plane0 != 0, row / batch sub-ranges, more tiles than SMs; both precisions.
  residual  P8 convs with a residual (GFF.1 <96,3>, the LFF's <96,1>): the epilogue loads all of a row's residual values
            before its first store.  res_plane0 / out_plane0 != 0, store_planes, sub-ranges; both precisions.
  final     UPNet.2 <16,3> + mean(frames): the frames are loaded before the main loop.  2, 3 and 5 frames, 1-3 calls,
            shared frame pools, both kernel variants, both precisions for the x-stacked one.
  convlstm  the forward cell at a vector-path (W % 4 == 0) and a scalar-path width, with and without state, at sizes
            with many more blocks than SMs; 1, 2 and 3 cells per launch, each cell of a group with the bits of its own
            one-cell launch.

Every tensor plane a call does not read holds NaN, every output element it must not write holds a sentinel, and both
keep their bits.  Bars as in test_gpu_forward_fuzz.py (u = 2^-24, A = fp64 conv of absolute values):
  fp16    |got - ref| <= ulp16(ref) + 32 u A                                ref: fp64 on the same fp16 operands
  X3      |got - ref| <= 32 u (A + |res|) + 2^-22 (3 A + |ref| + 2 |res|) + 2^-25 (W1 + 2) + 2^-33 X1   (fp32 operands)
  FINAL   the above without the output split, plus ulp32(ref) + (n + 1) u sum_f |frame_f|
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
SENTINEL = -1234.0
U = 2.0 ** -24
C_BAR = 32.0


def ulp16(v):
    return torch.exp2(torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -14))) - 10)


def ulp32(v):
    return torch.exp2(torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -126))) - 23)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


def _x3_plane(lp):
    return 2 * (lp & ~3) + (lp & 3)


def _to_device(vals, x3):
    """fp64 (B, 8 planes, H, W) -> P8 fp16 [B, planes, H, W, 8], or its (hi, lo) layout for x3."""
    B, C8, H, W = vals.shape
    p8 = vals.view(B, C8 // 8, 8, H, W).permute(0, 1, 3, 4, 2).float()
    if not x3:
        return p8.half().contiguous()
    hi = p8.half()
    lo = (p8 - hi.float()).half()
    out = torch.empty((B, 2 * (C8 // 8), H, W, 8), dtype=torch.float16, device=DEV)
    for lp in range(C8 // 8):
        out[:, _x3_plane(lp)] = hi[:, lp]
        out[:, _x3_plane(lp) + 4] = lo[:, lp]
    return out


def _from_device(t, plane0, n, x3):
    if x3:
        idx = torch.tensor([_x3_plane(lp) for lp in range(plane0, plane0 + n)], device=DEV)
        v = t[:, idx].double() + t[:, idx + 4].double()
    else:
        v = t[:, plane0:plane0 + n].double()
    B, _, H, W, _ = v.shape
    return v.permute(0, 1, 4, 2, 3).reshape(B, 8 * n, H, W)


def _phys(plane0, n, x3):
    lps = range(plane0, plane0 + n)
    return sorted([_x3_plane(p) for p in lps] + [_x3_plane(p) + 4 for p in lps]) if x3 else list(lps)


def _unchanged(t, before, planes, bsl, ysl, where):
    """Everything of t outside planes x batches bsl x rows ysl keeps its bits."""
    keep = torch.ones(t.shape, dtype=torch.bool, device=DEV)
    m = torch.zeros(t.shape, dtype=torch.bool, device=DEV)
    m[bsl, :, ysl] = True
    pm = torch.zeros(t.shape[1], dtype=torch.bool, device=DEV)
    pm[torch.tensor(planes, dtype=torch.long, device=DEV)] = True
    keep &= ~(m & pm.view(1, -1, 1, 1, 1))
    assert torch.equal(_bits(t)[keep], _bits(before)[keep]), ("wrote outside its range", where)


def _sub(sub, B, H):
    b0, nb, y0, ny = sub if sub else (0, B, 0, H)
    return slice(b0, b0 + nb), slice(y0, y0 + ny)


def _conv_bar(ref, A, W1, X1, x3, rabs=0.0):
    if x3:
        return C_BAR * U * (A + rabs) + 2.0 ** -22 * (3 * A + ref.abs() + 2 * rabs) + 2.0 ** -25 * (W1 + 2) + 2.0 ** -33 * X1
    return ulp16(ref) + C_BAR * U * A


def _weights(gen, cout, cin, k, x3, cout_pad, variant=0):
    from bin_b200 import ops
    rn = lambda *s: torch.randn(s, generator=gen, device=DEV, dtype=torch.float64)
    w32 = (rn(cout, cin, k, k) / math.sqrt(cin * k * k)).float()
    b32 = (rn(cout) * 0.1).float()
    opnd = (lambda t: t.float().double()) if x3 else (lambda t: t.half().double())
    wpad = torch.zeros((cout_pad, cin, k, k), dtype=torch.float64, device=DEV)
    wpad[:cout] = opnd(w32)
    bpad = torch.zeros(cout_pad, dtype=torch.float64, device=DEV)
    bpad[:cout] = b32.double()
    return ops.pack_conv_weight(w32, cout_pad, cin, variant=variant, prec=int(x3)), ops.pad_bias(b32, cout_pad), wpad, bpad


def _input(gen, B, planes, H, W, plane0, nplanes, x3, mag=1.0):
    """fp64 tensor of `planes` planes, NaN except planes [plane0, +nplanes) which hold the operands the kernel sees."""
    v = torch.full((B, 8 * planes, H, W), NAN, dtype=torch.float64, device=DEV)
    x = torch.randn((B, 8 * nplanes, H, W), generator=gen, device=DEV, dtype=torch.float64) * mag
    v[:, 8 * plane0:8 * (plane0 + nplanes)] = x.float().double() if x3 else x.half().double()
    return v


# --------------------------------------------------------------------------------------------------------------------
# UPNet.0 + PixelShuffle(2)
# --------------------------------------------------------------------------------------------------------------------
PIXSHUF = [  # (B, H, W, sub, in_plane0, out_plane0, x3)
    (1, 13, 47, None, 0, 8, False), (3, 9, 61, None, 4, 16, False), (2, 17, 95, (1, 1, 3, 11), 0, 8, False),
    (3, 45, 121, None, 0, 8, False), (1, 1, 1, None, 0, 0, False), (3, 7, 31, None, 4, 8, True),
    (2, 11, 89, (0, 2, 2, 7), 0, 16, True), (3, 21, 62, None, 0, 8, True),
]


@pytest.mark.parametrize("idx", range(len(PIXSHUF)))
def test_pixshuf_vs_fp64(idx):
    from bin_b200 import _lib, ops
    B, H, W, sub, ip0, op0, x3 = PIXSHUF[idx]
    where = PIXSHUF[idx]
    gen = torch.Generator(device=DEV).manual_seed(700 + idx)
    xin = _input(gen, B, ip0 + 12, H, W, ip0, 12, x3)
    X = xin[:, 8 * ip0:]
    outv = torch.full((B, 8 * (op0 + 12), 2 * H, 2 * W), NAN, dtype=torch.float64, device=DEV)
    outv[:, 8 * op0:8 * (op0 + 8)] = SENTINEL
    din, dout = _to_device(xin, x3), _to_device(outv, x3)
    before_in, before_out = din.clone(), dout.clone()
    wp, bp, w64, b64 = _weights(gen, 256, 96, 3, x3, 256)
    ops.conv_fwd(din, wp, bp, 3, 256, in0_plane0=ip0, in0_planes=12, epilogue=_lib.EPI_PIXSHUF, out=dout,
                 out_plane0=op0, sub=sub, x3=x3)
    torch.cuda.synchronize()
    ref = F.pixel_shuffle(F.conv2d(X, w64, b64, padding=1), 2)
    A = F.pixel_shuffle(F.conv2d(X.abs(), w64.abs(), b64.abs(), padding=1), 2)
    W1 = w64.abs().sum((1, 2, 3)).max()
    X1 = F.conv2d(X.abs(), torch.ones((1, 96, 3, 3), dtype=torch.float64, device=DEV), padding=1)
    X1 = X1.repeat_interleave(2, 2).repeat_interleave(2, 3)
    bar = _conv_bar(ref, A, W1, X1, x3)
    bsl, ysl = _sub(sub, B, H)
    ysl2 = slice(2 * ysl.start, 2 * ysl.stop)
    got = _from_device(dout, op0, 8, x3)
    assert torch.isfinite(got[bsl, :, ysl2]).all(), where
    ratio = ((got - ref)[bsl, :, ysl2].abs() / bar[bsl, :, ysl2]).max().item()
    assert ratio <= 1.0, (where, ratio)
    _unchanged(dout, before_out, _phys(op0, 8, x3), bsl, ysl2, where)
    assert torch.equal(_bits(din), _bits(before_in)), where


# --------------------------------------------------------------------------------------------------------------------
# P8 convs with a residual (GFF.1, LFF)
# --------------------------------------------------------------------------------------------------------------------
RESIDUAL = [  # (k, B, H, W, sub, res_plane0, out_plane0, store_planes, x3)
    (3, 2, 13, 47, None, 4, 8, 0, False), (3, 3, 9, 95, (1, 2, 1, 7), 0, 0, 8, False),
    (3, 3, 45, 121, None, 0, 12, 0, False), (3, 1, 1, 1, None, 4, 4, 0, False), (1, 2, 10, 37, None, 4, 0, 0, False),
    (3, 2, 11, 61, None, 4, 12, 0, True), (3, 3, 17, 31, (0, 3, 5, 9), 0, 4, 8, True), (1, 3, 7, 65, None, 8, 4, 0, True),
]


@pytest.mark.parametrize("idx", range(len(RESIDUAL)))
def test_residual_vs_fp64(idx):
    from bin_b200 import ops
    k, B, H, W, sub, rp0, op0, store, x3 = RESIDUAL[idx]
    where = RESIDUAL[idx]
    gen = torch.Generator(device=DEV).manual_seed(800 + idx)
    nstore = store or 12
    X_v = _input(gen, B, 12, H, W, 0, 12, x3)
    res_v = _input(gen, B, rp0 + 12, H, W, rp0, nstore, x3)
    out_v = torch.full((B, 8 * (op0 + 12), H, W), NAN, dtype=torch.float64, device=DEV)
    out_v[:, 8 * op0:8 * (op0 + nstore)] = SENTINEL
    dx, dres, dout = _to_device(X_v, x3), _to_device(res_v, x3), _to_device(out_v, x3)
    before = [dx.clone(), dres.clone(), dout.clone()]
    wp, bp, w64, b64 = _weights(gen, 96, 96, k, x3, 96)
    ops.conv_fwd(dx, wp, bp, k, 96, in0_planes=12, out=dout, out_plane0=op0, res=dres, res_plane0=rp0, sub=sub,
                 store_planes=store, x3=x3)
    torch.cuda.synchronize()
    r = res_v[:, 8 * rp0:8 * (rp0 + nstore)]
    ref = F.conv2d(X_v, w64, b64, padding=k // 2)[:, :8 * nstore] + r
    A = F.conv2d(X_v.abs(), w64.abs(), b64.abs(), padding=k // 2)[:, :8 * nstore]
    W1 = w64.abs().sum((1, 2, 3)).view(1, -1, 1, 1)[:, :8 * nstore]
    X1 = F.conv2d(X_v.abs(), torch.ones((1, 96, k, k), dtype=torch.float64, device=DEV), padding=k // 2)
    bar = _conv_bar(ref, A, W1, X1, x3, r.abs())
    bsl, ysl = _sub(sub, B, H)
    got = _from_device(dout, op0, nstore, x3)
    assert torch.isfinite(got[bsl, :, ysl]).all(), where
    ratio = ((got - ref)[bsl, :, ysl].abs() / bar[bsl, :, ysl]).max().item()
    assert ratio <= 1.0, (where, ratio)
    _unchanged(dout, before[2], _phys(op0, nstore, x3), bsl, ysl, where)
    assert torch.equal(_bits(dx), _bits(before[0])) and torch.equal(_bits(dres), _bits(before[1])), where


# --------------------------------------------------------------------------------------------------------------------
# UPNet.2 + mean(frames)
# --------------------------------------------------------------------------------------------------------------------
FINAL = [  # (nframes, ncalls, Bc, shared, H, W, sub, variant, x3)
    (2, 1, 1, False, 13, 47, None, 0, False), (3, 2, 1, True, 9, 61, None, 0, False),
    (5, 3, 1, True, 17, 95, (1, 2, 3, 11), 0, False), (5, 2, 2, False, 45, 121, None, 0, False),
    (2, 3, 1, True, 7, 31, None, 1, False), (3, 1, 3, False, 11, 89, (0, 2, 2, 7), 1, False),
    (5, 2, 1, True, 21, 62, None, 1, False),
    (2, 2, 1, False, 11, 61, None, 0, True), (3, 1, 2, True, 9, 47, (1, 1, 0, 5), 0, True), (5, 3, 1, True, 13, 35, None, 0, True),
]


@pytest.mark.parametrize("idx", range(len(FINAL)))
def test_final_vs_fp64(idx):
    from bin_b200 import _lib, ops
    nf, nc, Bc, shared, H, W, sub, variant, x3 = FINAL[idx]
    where = FINAL[idx]
    B = nc * Bc
    gen = torch.Generator(device=DEV).manual_seed(900 + idx)
    X_v = _input(gen, B, 8, H, W, 0, 8, x3)
    dx = _to_device(X_v, x3)
    before = dx.clone()
    wp, bp, w64, b64 = _weights(gen, 3, 64, 3, x3, 16, variant)
    npool = nc * (nf - 1) + 1 if shared else nc * nf
    pool = [torch.rand((Bc, 3, H, W), generator=gen, device=DEV) for _ in range(npool)]
    frames = [[pool[c * (nf - 1) + f] if shared else pool[c * nf + f] for f in range(nf)] for c in range(nc)]
    outs = [torch.full((Bc, 3, H, W), SENTINEL, device=DEV) for _ in range(nc)]
    outs0 = [o.clone() for o in outs]
    table = ops.make_frames(frames, outs)
    ops.conv_fwd(dx, wp, bp, 3, 16, in0_planes=8, epilogue=_lib.EPI_FINAL, frames=table, variant=variant, sub=sub, x3=x3)
    torch.cuda.synchronize()
    conv = F.conv2d(X_v, w64, b64, padding=1)[:, :3]
    A = F.conv2d(X_v.abs(), w64.abs(), b64.abs(), padding=1)[:, :3]
    W1 = w64.abs().sum((1, 2, 3)).view(1, -1, 1, 1)[:, :3]
    X1 = F.conv2d(X_v.abs(), torch.ones((1, 64, 3, 3), dtype=torch.float64, device=DEV), padding=1)
    fsum = torch.cat([sum(f.double() for f in fr) for fr in frames], 0)
    fabs = torch.cat([sum(f.double().abs() for f in fr) for fr in frames], 0)
    ref = conv + fsum / nf
    extra = ulp32(ref) + (nf + 1) * U * fabs
    bar = (C_BAR * U * A + 2.0 ** -22 * 3 * A + 2.0 ** -25 * W1 + 2.0 ** -33 * X1 if x3 else C_BAR * U * A) + extra
    got = torch.cat([o.double() for o in outs], 0)
    bsl, ysl = _sub(sub, B, H)
    assert torch.isfinite(got[bsl, :, ysl]).all(), where
    ratio = ((got - ref)[bsl, :, ysl].abs() / bar[bsl, :, ysl]).max().item()
    assert ratio <= 1.0, (where, ratio)
    for c, (o, o0) in enumerate(zip(outs, outs0)):
        m = torch.ones(o.shape, dtype=torch.bool, device=DEV)
        for bb in range(Bc):
            if bsl.start <= c * Bc + bb < bsl.stop:
                m[bb, :, ysl] = False
        assert torch.equal(_bits(o)[m], _bits(o0)[m]), ("final wrote outside its range", c, where)
    assert torch.equal(_bits(dx), _bits(before)), where
    del table


# --------------------------------------------------------------------------------------------------------------------
# ConvLSTM cell
# --------------------------------------------------------------------------------------------------------------------
K_LSTM, T_LSTM = 56.0, 3e-7


def _convlstm_launch(cells, B, H, W):
    """One bin_convlstm_fwd launch over the cell table [(x, w, b, c_prev, h_prev), ...] -> ([h], [c]), NaN-filled first."""
    from bin_b200 import _lib
    P = lambda t: None if t is None else t.data_ptr()
    hs = [torch.full((B, 3, H, W), NAN, device=DEV) for _ in cells]
    cs = [torch.full((B, 3, H, W), NAN, device=DEV) for _ in cells]
    tab = (_lib.LstmCell * len(cells))(*[_lib.LstmCell(x.data_ptr(), P(cp), P(hp), w.data_ptr(), b.data_ptr(), h.data_ptr(),
                                                       c.data_ptr()) for (x, w, b, cp, hp), h, c in zip(cells, hs, cs)])
    _lib.check(_lib.lib().bin_convlstm_fwd(tab, len(cells), B, H, W, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return hs, cs


@pytest.mark.parametrize("ncells", [1, 2, 3])
@pytest.mark.parametrize("state", [False, True])
@pytest.mark.parametrize("W", [1280, 1283])
def test_convlstm_large_vs_fp64(W, state, ncells):
    """ncells cells with their own inputs and weights in one launch: every cell against fp64, and with more than one
    cell every cell with the bits of its own one-cell launch."""
    B, H = 2, 37
    gen = torch.Generator(device=DEV).manual_seed(1000 + W + int(state))
    cells = []
    for _ in range(ncells):
        x = torch.randn((B, 3, H, W), generator=gen, device=DEV) * 3
        w = torch.randn((12, 6, 3, 3), generator=gen, device=DEV) * 2
        b = torch.randn((12,), generator=gen, device=DEV)
        cp = (torch.rand((B, 3, H, W), generator=gen, device=DEV) * 100 - 50) if state else None
        hp = (torch.rand((B, 3, H, W), generator=gen, device=DEV) * 2 - 1) if state else None
        cells.append((x, w, b, cp, hp))
    hs, cs = _convlstm_launch(cells, B, H, W)
    for k, ((x, w, b, cp, hp), h, c) in enumerate(zip(cells, hs, cs)):
        c0 = cp.double() if state else torch.zeros((B, 3, H, W), dtype=torch.float64, device=DEV)
        h0 = hp.double() if state else torch.zeros_like(c0)
        xh = torch.cat((x.double(), h0), 1)
        gi, gj, gf, go = F.conv2d(xh, w.double(), b.double(), padding=1).chunk(4, 1)
        Gi, Gj, Gf, Go = F.conv2d(xh.abs(), w.double().abs(), b.double().abs(), padding=1).chunk(4, 1)
        si, tj, sf, so = torch.sigmoid(gi), torch.tanh(gj), torch.sigmoid(gf + 1.0), torch.sigmoid(go)
        c_ref = c0 * sf + si * tj
        h_ref = torch.tanh(c_ref) * so
        e_i, e_f, e_o = (0.25 * K_LSTM * U * G_ + T_LSTM for G_ in (Gi, Gf + 1.0, Go))
        e_j = K_LSTM * U * Gj + T_LSTM
        e_c = c0.abs() * e_f + tj.abs() * e_i + si.abs() * e_j + 3 * U * (c0 * sf).abs() + 3 * U * (si * tj).abs()
        e_h = so.abs() * (e_c + T_LSTM) + torch.tanh(c_ref).abs() * e_o + U * h_ref.abs()
        assert ((h.double() - h_ref).abs() / e_h).max().item() <= 1.0, k
        assert ((c.double() - c_ref).abs() / e_c).max().item() <= 1.0, k
        if ncells > 1:
            (h1,), (c1,) = _convlstm_launch([cells[k]], B, H, W)
            assert torch.equal(_bits(h), _bits(h1)) and torch.equal(_bits(c), _bits(c1)), k
