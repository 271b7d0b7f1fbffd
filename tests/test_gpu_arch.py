"""The backbone configurations G0 in {64, 96}, 1 <= D <= 12 on the GPU: the conv instantiations the G0 = 64 backbones add,
and the G0 = 96 layers whose tensors change with D, against fp64 per element; the G0 = 64 fused RDB tail against fp64
and bit for bit against its layer-by-layer path; every backbone class and the light window (net.model =
RDN_residual_interp_5_input(lstm=True, GO=64, D=6)) against the reference's fixtures (oracle/make_golden_arch.py) and the
oracle, with the shipped bars; the inference modes on a light window; per-tensor backbone gradients against fp64 at
the depth edges of both widths, and the training stack on a light window."""
import contextlib
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from no_flip import check_no_relu_near_zero, no_flip_sd, oracle_grads
from oracle import arch_oracle as A
from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
SENTINEL = -1234.0
U = 2.0 ** -24
C_F16, C_X3, C_TAIL = 32.0, 32.0, 32.0           # the bars of test_gpu_forward_fuzz.py
TOL_FP16, TOL_FP32_MODE, TOL_PSNR = 1e-3, 1e-5, 0.01
CLASSES = {2: "RDN_residual_interp_2_input", 3: "RDN_residual_interp_2_1_input", 5: "RDN_residual_interp_4_1_input"}


def ulp16(v):
    return torch.exp2(torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -14))) - 10)


def _x3_plane(lp):
    return 2 * (lp & ~3) + (lp & 3)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


def _to_device(vals, x3):
    """fp64 (B, 8 planes, H, W) -> P8 fp16, or its (hi, lo) layout for x3."""
    B, C8, H, W = vals.shape
    p8 = vals.view(B, C8 // 8, 8, H, W).permute(0, 1, 3, 4, 2).float()
    if not x3:
        return p8.half().contiguous()
    hi = p8.half()
    lo = (p8 - hi.float()).half()
    out = torch.empty((B, 2 * (C8 // 8), H, W, 8), dtype=torch.float16, device=vals.device)
    for lp in range(C8 // 8):
        out[:, _x3_plane(lp)], out[:, _x3_plane(lp) + 4] = hi[:, lp], lo[:, lp]
    return out


def _from_device(t, plane0, nplanes, x3):
    if x3:
        idx = torch.tensor([_x3_plane(lp) for lp in range(plane0, plane0 + nplanes)], device=t.device)
        v = t[:, idx].double() + t[:, idx + 4].double()
    else:
        v = t[:, plane0:plane0 + nplanes].double()
    B, _, H, W, _ = v.shape
    return v.permute(0, 1, 4, 2, 3).reshape(B, 8 * nplanes, H, W)


def _phys(plane0, n, x3):
    lps = range(plane0, plane0 + n)
    return sorted([_x3_plane(p) for p in lps] + [_x3_plane(p) + 4 for p in lps]) if x3 else list(lps)


# --------------------------------------------------------------------------------------------------------------------
# part 1: the G0 = 64 conv instantiations <64,5>, <64,3>, <64,1> against fp64, both precisions, and the G0 = 96 layers
# whose tensors change with D
# --------------------------------------------------------------------------------------------------------------------
def _layer(kind, g0=64, d=6, i=3, train=False):
    """(k, cin, tensors {name: planes}, segs [(tensor, plane0, planes)], out (tensor, plane0), res) as a backbone of
    width g0 (P = g0 / 8 planes per feature map) launches the layer: SFENet1 on the packed frames, SFENet2, GFF.1 with
    f1, the LFF of RDB i (x = cat[P(i-1), +P) or f2, g at 16 i when training, output cat[P i]), GFF.0 on the D x
    g0-channel concat."""
    P = g0 // 8
    if kind.startswith("sfe1"):
        cin = int(kind[4:])
        xp = (cin + 31) // 32 * 4
        return 5, cin, dict(x0=xp, f1=P), [("x0", 0, xp)], ("f1", 0), None
    if kind == "sfe2":
        return 3, g0, dict(f1=2 * P, f2=P), [("f1", 4, P)], ("f2", 0), None
    if kind == "gff1":
        return 3, g0, dict(t1=P, t2=P, f1=P), [("t1", 0, P)], ("t2", 0), ("f1", 0)
    if kind == "lff":
        gp0 = 16 * i if train else 0
        x = ("cat", P * (i - 1), P) if i else ("f2", 0, P)
        tensors = dict(g=16 * d if train else 16, cat=P * d, f2=P)
        return 1, g0 + 128, tensors, [x, ("g", gp0, 16)], ("cat", P * i), x[:2]
    if kind == "gff0":
        return 1, g0 * d, dict(cat=P * d, t1=P), [("cat", 0, P * d)], ("t1", 0), None
    raise ValueError(kind)


MANY = (3, 72, 130)                   # more tiles than SMs for every kernel
CONV_CASES = {  # name: (layer kind, layer options, B, H, W, sub, magnitude)
    "sfe1_24": ("sfe124", {}, 2, 9, 27, None, 1.0),
    "sfe1_36_sub": ("sfe136", {}, 3, 17, 57, (1, 1, 4, 9), 2.0 ** 5),
    "sfe1_60_many": ("sfe160", {}, *MANY, None, 1.0),
    "sfe2": ("sfe2", {}, 2, 16, 61, None, 1.0),
    "sfe2_1x1": ("sfe2", {}, 3, 1, 1, None, 2.0 ** -12),
    "sfe2_many": ("sfe2", {}, *MANY, None, 1.0),
    "gff1_res_sub": ("gff1", {}, 3, 16, 61, (0, 2, 7, 8), 1.0),
    "gff1_many": ("gff1", {}, *MANY, None, 1.0),
    "lff_i0": ("lff", dict(i=0), 2, 9, 31, None, 1.0),
    "lff_i5_train": ("lff", dict(i=5, train=True), 2, 16, 33, None, 1.0),
    "lff_i11_train_d12_sub": ("lff", dict(i=11, d=12, train=True), 1, 7, 32, (0, 1, 2, 3), 2.0 ** -12),
    "lff_many": ("lff", dict(i=2), *MANY, None, 1.0),
    "gff0_d1": ("gff0", dict(d=1), 2, 9, 33, None, 1.0),
    "gff0_d6": ("gff0", dict(d=6), 2, 7, 1, None, 1.0),
    "gff0_d12_many": ("gff0", dict(d=12), *MANY, None, 1.0),
}
# G0 = 96 (the <96,k> kernels): GFF.0 reads D x 12 planes, and the LFF of the last RDB writes the last 12 planes of cat
CONV_CASES_G96 = {
    "g96_gff0_d1": ("gff0", dict(g0=96, d=1), 2, 9, 33, None, 1.0),
    "g96_gff0_d3": ("gff0", dict(g0=96, d=3), 3, 11, 47, (1, 2, 3, 7), 1.0),
    "g96_gff0_d5": ("gff0", dict(g0=96, d=5), 1, 16, 61, None, 2.0 ** 5),
    "g96_lff_last_d1": ("lff", dict(g0=96, d=1, i=0), 2, 9, 31, None, 1.0),
    "g96_lff_last_d5_train": ("lff", dict(g0=96, d=5, i=4, train=True), 2, 15, 34, None, 1.0),
}


@pytest.mark.parametrize("x3", [False, True])
@pytest.mark.parametrize("case", sorted(CONV_CASES) + sorted(CONV_CASES_G96))
def test_g64_conv_vs_fp64(case, x3):
    """NaN in every plane the call must not read, the sentinel in every element it must not write; per-element bars of
    test_gpu_forward_fuzz.py (fp16: ulp16(ref) + 32 u A; x3: the split-operand bar)."""
    from bin_b200 import ops
    if case in CONV_CASES:
        kind, opts, B, H, W, sub, mag = CONV_CASES[case]
        seed = 2 * sorted(CONV_CASES).index(case) + int(x3)
    else:
        kind, opts, B, H, W, sub, mag = CONV_CASES_G96[case]
        seed = 1000 + 2 * sorted(CONV_CASES_G96).index(case) + int(x3)
    g0 = opts.get("g0", 64)
    k, cin, tensors, segs, (on, op0), res = _layer(kind, **opts)
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *shape: torch.randn(shape, generator=g, device=DEV, dtype=torch.float64)
    opnd = (lambda t: t.float().double()) if x3 else (lambda t: t.half().double())
    vals = {n: torch.full((B, 8 * p, H, W), NAN, dtype=torch.float64, device=DEV) for n, p in tensors.items()}
    for name, p0, np_ in list(segs) + ([(res[0], res[1], g0 // 8)] if res else []):
        blk = vals[name][:, 8 * p0:8 * (p0 + np_)]
        fill = torch.isnan(blk)
        blk[fill] = opnd(rn(*blk.shape) * mag)[fill]
    X = torch.cat([vals[n][:, 8 * p0:8 * (p0 + np_)] for n, p0, np_ in segs], 1)
    if X.shape[1] > cin:                                  # SFENet1: the packer's zero channels past 12 n
        X[:, cin:] = 0
        vals[segs[0][0]][:, cin:] = 0
    if res is not None and res[0] == on:
        assert res[1] != op0
    vals[on][:, 8 * op0:8 * op0 + g0] = SENTINEL
    dev_t = {n: _to_device(v, x3) for n, v in vals.items()}
    before = {n: t.clone() for n, t in dev_t.items()}
    w32 = (rn(g0, X.shape[1], k, k) / math.sqrt(cin * k * k)).float()
    w32[:, cin:] = 0
    b32 = (rn(g0) * 0.1 * mag).float()
    kw = dict(in0_plane0=segs[0][1], in0_planes=segs[0][2], sub=sub, x3=x3, out=dev_t[on], out_plane0=op0)
    if len(segs) > 1:
        kw.update(in1=dev_t[segs[1][0]], in1_plane0=segs[1][1], in1_planes=segs[1][2])
    if res:
        kw.update(res=dev_t[res[0]], res_plane0=res[1])
    ops.conv_fwd(dev_t[segs[0][0]], ops.pack_conv_weight(w32, g0, X.shape[1], prec=int(x3)), ops.pad_bias(b32, g0), k, g0,
                 **kw)
    torch.cuda.synchronize()
    w64, b64 = opnd(w32), b32.double()
    ref = F.conv2d(X, w64, b64, padding=k // 2)
    A = F.conv2d(X.abs(), w64.abs(), b64.abs(), padding=k // 2)
    rabs = 0.0
    if res:
        r = vals[res[0]][:, 8 * res[1]:8 * res[1] + g0]
        ref, rabs = ref + r, r.abs()
    if x3:
        W1 = w64.abs().sum((1, 2, 3)).view(1, -1, 1, 1)
        X1 = F.conv2d(X.abs(), torch.ones((1,) + w64.shape[1:], dtype=torch.float64, device=DEV), padding=k // 2)
        bar = C_X3 * U * (A + rabs) + 2.0 ** -22 * (3 * A + ref.abs() + 2 * rabs) + 2.0 ** -25 * (W1 + 2) + 2.0 ** -33 * X1
    else:
        bar = ulp16(ref) + C_F16 * U * A
    got = _from_device(dev_t[on], op0, g0 // 8, x3)
    b0, nb, y0, ny = sub if sub else (0, B, 0, H)
    sl = (slice(b0, b0 + nb), slice(None), slice(y0, y0 + ny))
    assert torch.isfinite(got[sl]).all(), case
    ratio = ((got - ref)[sl].abs() / bar[sl]).max().item()
    print(f"[conv G0={g0}] {case} {'x3' if x3 else 'f16'}: worst err/bar {ratio:.3f}")
    assert ratio <= 1.0, (case, x3, ratio)
    for name, t in dev_t.items():
        keep = torch.ones(t.shape, dtype=torch.bool, device=DEV)
        if name == on:
            pm = torch.zeros(t.shape[1], dtype=torch.bool, device=DEV)
            pm[torch.tensor(_phys(op0, g0 // 8, x3), device=DEV)] = True
            m = torch.zeros(t.shape, dtype=torch.bool, device=DEV)
            m[sl[0], :, sl[2]] = True
            keep &= ~(m & pm.view(1, -1, 1, 1, 1))
        assert torch.equal(_bits(t)[keep], _bits(before[name])[keep]), ("wrote outside its range", name, case)


# --------------------------------------------------------------------------------------------------------------------
# part 2: the G0 = 64 fused RDB tail
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,h,w", [(1, 4, 30), (2, 9, 37), (3, 17, 61), (1, 1, 1), (4, 120, 200)])
def test_g64_fused_tail_bit_identical_to_layerwise_and_vs_fp64(B, h, w):
    """bin_rdb_fwd on a G0 = 64 blob runs conv3 + LFF as the fused tail (rdb_tail_kernel<64>); RDB.forward runs the same
    four growth convs and the LFF as separate launches.  Same accumulation order: the same bits.  Both are held to fp64
    on the growth maps the kernels computed, with the tail bar of test_gpu_forward_fuzz.py."""
    import ctypes as C
    from bin_b200 import _lib, ops, rdn
    torch.manual_seed(h * 1000 + w)
    m = rdn.RDN_residual_interp_2_input(G0=64, D=2).cuda()
    blk = m.RDBs[1]
    gen = torch.Generator(device=DEV).manual_seed(B * 7 + h)
    with torch.no_grad():
        for p in blk.parameters():
            p.add_(torch.randn(p.shape, generator=gen, device=DEV) * 0.02)
    x = torch.randn((B, 64, h, w), generator=gen, device=DEV)
    L = _lib.lib()
    ws = torch.empty(B * 40 * h * w * 16 + 4096, dtype=torch.uint8, device=DEV)
    y = torch.empty_like(x)
    _lib.check(L.bin_rdb_fwd(m.packed_blob(0).data_ptr(), m.arch, 1, x.data_ptr(), y.data_ptr(), B, h, w, ws.data_ptr(),
                             ws.numel(), ops._stream()))
    with torch.no_grad():
        y_layer = blk(x)
    torch.cuda.synchronize()
    assert torch.equal(_bits(y), _bits(y_layer))
    # fp64 reference of the tail on the operands it read: x and g0..g2 in fp16, as the layer path computed them
    xin = ops.nchw_to_p8(x)
    g = ops.empty_p8(B, 16, h, w, DEV)
    for c in range(3):
        conv = blk.convs[c].conv[0]
        ops.conv_fwd(xin, ops.pack_conv_weight(conv.weight.detach(), 32, 64 + 32 * c), ops.pad_bias(conv.bias.detach(), 32),
                     3, 32, in0_planes=8, in1=g, in1_planes=4 * c, relu=True, out=g, out_plane0=4 * c)
    xd, g012 = _from_device(xin, 0, 8, False), _from_device(g, 0, 12, False)
    w3 = blk.convs[3].conv[0].weight.detach().half().double()
    b3 = blk.convs[3].conv[0].bias.detach().double()
    wl, bl = blk.LFF.weight.detach().half().double(), blk.LFF.bias.detach().double()
    in3 = torch.cat((xd, g012), 1)
    g3 = F.conv2d(in3, w3, b3, padding=1).relu().half().double()
    A3 = F.conv2d(in3.abs(), w3.abs(), b3.abs(), padding=1)
    inl = torch.cat((xd, g012, g3), 1)
    ref = F.conv2d(inl, wl, bl) + xd
    A = F.conv2d(inl.abs(), wl.abs(), bl.abs()) + xd.abs()
    # the kernel stores x' in fp16, which y reads back exactly
    bar = ulp16(ref) + C_F16 * U * A + F.conv2d(ulp16(g3) + C_TAIL * U * A3, wl[:, 160:].abs())
    ratio = ((y.double() - ref).abs() / bar).max().item()
    print(f"[g64 tail] B={B} {h}x{w}: worst err/bar {ratio:.3f}")
    assert ratio <= 1.0, ratio


# --------------------------------------------------------------------------------------------------------------------
# part 3: forward parity of every backbone class and of the light window
# --------------------------------------------------------------------------------------------------------------------
def _seed(n, g0, d):                      # oracle/make_golden_arch.py
    return 500 + 100 * n + g0 + d


def _backbone(n, g0, d, seed, precision="fp16"):
    from bin_b200 import rdn
    m = getattr(rdn, CLASSES[n])(G0=g0, D=d)
    m.load_state_dict(A.synth_backbone_sd(n, seed, g0, d), strict=True)
    return rdn.set_precision(m.cuda().eval(), precision)


@pytest.mark.parametrize("precision,bar", [("fp16", TOL_FP16), ("fp32", TOL_FP32_MODE)])
@pytest.mark.parametrize("g0,d", [(64, 6), (64, 12), (96, 6)])
@pytest.mark.parametrize("n", sorted(CLASSES))
def test_backbone_matches_reference_fixture(golden_dir, n, g0, d, precision, bar):
    g = np.load(os.path.join(golden_dir, "arch_backbones.npz"))
    B, H, W = [int(v) for v in g["meta"]]
    m = _backbone(n, g0, d, _seed(n, g0, d), precision)
    fr = O.synth_frames(n, B, H, W, seed=_seed(n, g0, d) + 1)
    with torch.no_grad():
        out = m(*[f.cuda() for f in fr]).cpu()
    err = (out - torch.from_numpy(g[f"{n}_{g0}_{d}"])).abs().max().item()
    assert err <= bar, (n, g0, d, precision, err)


@pytest.mark.parametrize("precision,bar", [("fp16", TOL_FP16), ("fp32", TOL_FP32_MODE)])
@pytest.mark.parametrize("g0,d", [(64, 1), (96, 1), (64, 3)])
@pytest.mark.parametrize("n", sorted(CLASSES))
def test_shallow_backbone_vs_oracle(n, g0, d, precision, bar):
    m = _backbone(n, g0, d, 77 + n, precision)
    fr = O.synth_frames(n, 2, 34, 62, seed=n)
    ref = A.backbone(fr, A.synth_backbone_sd(n, 77 + n, g0, d))
    with torch.no_grad():
        out = m(*[f.cuda() for f in fr]).cpu()
    assert (out - ref).abs().max().item() <= bar


def _light_net(precision="fp16", g0=64, d=6, seed=0):
    from bin_b200 import rdn
    net = rdn.bin_stage4_lstm()
    net.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=g0, D=d)
    net.load_state_dict(A.synth_state_dict(seed, g0, d), strict=True)
    return rdn.set_precision(net.cuda().eval(), precision)


@pytest.fixture(scope="module")
def light():
    return _light_net()


def _oracle_on_gpu(frames, sd, dtype=torch.float64):
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            out = A.window_forward([f.to(DEV, dtype) for f in frames], {k: v.to(DEV, dtype) for k, v in sd.items()})
            return [o.float() for o in out]
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


def _psnr_delta(got, ref, gt):
    p_ref = O.psnr_u8(O.tensor2img_u8(ref), O.tensor2img_u8(gt))
    p_got = O.psnr_u8(O.tensor2img_u8(got), O.tensor2img_u8(gt))
    return abs(p_ref - p_got)


@pytest.mark.parametrize("precision,bar", [("fp16", TOL_FP16), ("fp32", TOL_FP32_MODE)])
def test_light_window_matches_reference_fixture(golden_dir, precision, bar):
    g = np.load(os.path.join(golden_dir, "arch_window.npz"))
    B, H, W, seed, _ = [int(v) for v in g["meta"]]
    net = _light_net(precision)
    with torch.no_grad():
        outs = net(*[f.cuda() for f in O.synth_frames(6, B, H, W, seed=seed)])
    for k, o in enumerate(outs):
        err = (o.cpu() - torch.from_numpy(g[f"out{k}"])).abs().max().item()
        assert err <= bar, (k, precision, err)


@pytest.mark.parametrize("d,H,W", [(1, 64, 96), (12, 64, 96), (6, 720, 1280)])
def test_light_window_vs_oracle_and_psnr(d, H, W):
    """Windows of depth 1, 12 and 6 (the last at 1280x720, the benchmarked size) against the fp64 oracle on the GPU."""
    sd = A.synth_state_dict(3, 64, d)
    fr = O.synth_frames(6, 1, H, W, seed=1234, smooth=True)
    gt = O.synth_frames(14, 1, H, W, seed=4321, smooth=True)
    ref = _oracle_on_gpu(fr, sd)
    frc = [f.cuda() for f in fr]
    for precision, bar in (("fp16", TOL_FP16), ("fp32", TOL_FP32_MODE)):
        net = _light_net(precision, 64, d, 3)
        with torch.no_grad():
            outs = net(*frc)
        worst = max((o - r).abs().max().item() for o, r in zip(outs, ref))
        print(f"[light window D={d} {W}x{H} {precision}] max-abs {worst:.3e}")
        assert worst <= bar, (precision, worst)
        if precision == "fp16":
            psnr = max(_psnr_delta(o.cpu(), r.cpu(), g_) for o, r, g_ in zip(outs, ref, gt))
            assert psnr <= TOL_PSNR, psnr
        del net, outs


# --------------------------------------------------------------------------------------------------------------------
# part 4: inference modes on the light window
# --------------------------------------------------------------------------------------------------------------------
def test_light_streaming_and_output_selection_keep_the_bits(light):
    from bin_b200 import rdn
    from bin_b200.streaming import StreamingBIN
    video = [f.cuda() for f in O.synth_frames(8, 1, 48, 80, seed=77, smooth=True)]
    st = StreamingBIN(light)
    got = [st.push(f) for f in video]
    with torch.no_grad():
        for k in range(3):
            ref = light(*video[k:k + 6])
            assert all(torch.equal(a, b) for a, b in zip(got[5 + k], ref)), k
        try:
            rdn.set_outputs(light, (13, 8, 12))
            sel = light(*video[:6])
        finally:
            rdn.set_outputs(light, None)
        full = light(*video[:6])
    for i in range(14):
        assert (sel[i] is None) if i not in (8, 12, 13) else torch.equal(sel[i], full[i]), i


def test_light_flipx4_matches_the_oracle_ensemble(light):
    from bin_b200 import rdn
    sd = A.synth_state_dict(0, 64, 6)
    fr = O.synth_frames(6, 1, 32, 48, seed=8, smooth=True)
    flips = [None, (-1,), (-2,), (-2, -1)]
    acc = None
    for dims in flips:
        outs = A.window_forward([f if dims is None else torch.flip(f, dims) for f in fr], sd)
        outs = [o if dims is None else torch.flip(o, dims) for o in outs]
        acc = outs if acc is None else [a + o for a, o in zip(acc, outs)]
    ref = [a / 4 for a in acc]
    try:
        rdn.set_self_ensemble(light, "flipx4")
        with torch.no_grad():
            got = light(*[f.cuda() for f in fr])
    finally:
        rdn.set_self_ensemble(light, None)
    assert max((g.cpu() - r).abs().max().item() for g, r in zip(got, ref)) <= TOL_FP16


# --------------------------------------------------------------------------------------------------------------------
# part 5: training
# --------------------------------------------------------------------------------------------------------------------
def _backbone_grads(model, pool, calls_idx, cots, mode=None, frozen=(), frame_grad=True):
    """One forward and backward of `model` on the calls, with activation checkpointing `mode`, the parameters whose names
    start with one of `frozen` at requires_grad False and the frames at requires_grad `frame_grad`: every parameter's
    and frame's gradient (None where none was asked for)."""
    from bin_b200 import autograd, rdn
    rdn.set_activation_checkpointing(model, mode)
    try:
        model.zero_grad(set_to_none=True)
        for k, p in model.named_parameters():
            p.requires_grad_(not k.startswith(frozen))
        frg = [p.cuda().requires_grad_(frame_grad) for p in pool]
        outs = autograd.backbone_stage(model, [[frg[j] for j in idx] for idx in calls_idx])
        sum((o * c.cuda()).sum() for o, c in zip(outs, cots)).backward()
        grads = {k: None if p.grad is None else p.grad.clone() for k, p in model.named_parameters()}
        grads.update({f"frame{j}": f.grad for j, f in enumerate(frg)})
        return grads
    finally:
        rdn.set_activation_checkpointing(model, None)
        for p in model.parameters():
            p.requires_grad_(True)


# (g0, d, n, ncalls, Bc, H, W, seed): G0 = 64, D = 6 keeps the ids and seeds it had as the only configuration; the depth
# edges D = 1 (RDB 0 is the first and the last RDB, d cat one G0 block), odd D (GFF.0's rows and channels end in
# partial blocks at G0 = 64) and D = 12 at G0 = 64 (d cat 96 planes, growth maps 192), the three backbone classes in turn
BWD_CASES = [
    pytest.param(64, 6, 2, 1, 2, 44, 68, 302, id="2-1-2-44-68"),
    pytest.param(64, 6, 3, 3, 1, 30, 50, 303, id="3-3-1-30-50"),
    pytest.param(64, 6, 5, 1, 1, 30, 50, 305, id="5-1-1-30-50"),
    pytest.param(64, 1, 2, 1, 2, 30, 50, 401, id="g64-d1-n2"),
    pytest.param(64, 5, 3, 1, 1, 30, 50, 402, id="g64-d5-n3"),
    pytest.param(64, 12, 5, 1, 1, 30, 50, 403, id="g64-d12-n5"),
    pytest.param(96, 1, 3, 3, 1, 30, 50, 404, id="g96-d1-n3-ncalls3"),
    pytest.param(96, 5, 5, 1, 2, 30, 50, 405, id="g96-d5-n5"),
    pytest.param(96, 6, 2, 1, 1, 44, 68, 406, id="g96-d6-n2"),
]


@pytest.mark.parametrize("g0,d,n,ncalls,Bc,H,W,seed", BWD_CASES)
def test_light_backbone_backward_without_relu_flips(g0, d, n, ncalls, Bc, H, W, seed):
    """The per-tensor gradient check of test_gpu_backward_fuzz.py at width g0 and depth d, with its bars: the forward
    within TOL_FP16; each gradient within 2x (4x for the bias of growth convs 0-2) the error an fp16-storage oracle
    makes, plus 1e-3 of the tensor's max; the "off" growth channels' weights and biases exactly 0.  Then, in
    deterministic mode, bit for bit: a second backward, the recomputing backward, and backwards with SFENet1 and RDB 0
    frozen (the need mask cuts both ends of the walk), with and without frame gradients."""
    from bin_b200 import autograd, rdn
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        pool = O.synth_frames(ncalls + max(n - 2, 1), Bc, H, W, seed=seed + 17 * ncalls + Bc)
        calls_idx = [list(range(k, k + n - 1)) + [k + 1] for k in range(ncalls)]
        cots = [c - 0.5 for c in O.synth_frames(ncalls, Bc, H, W, seed=seed + 1)]
        pool64 = [p.to(DEV, torch.float64) for p in pool]
        sd = {k: v.cpu() for k, v in no_flip_sd(n, seed, [[pool64[j] for j in idx] for idx in calls_idx], g0, d).items()}
        check_no_relu_near_zero([[pool64[j] for j in idx] for idx in calls_idx], sd, min_cv=None)
        ref_outs, gfr, gp = oracle_grads(pool, calls_idx, cots, sd, emulate=False)
        _, gfr_emu, gp_emu = oracle_grads(pool, calls_idx, cots, sd, emulate=True)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    model = getattr(rdn, CLASSES[n])(G0=g0, D=d)
    model.load_state_dict(sd, strict=True)
    model = model.cuda()
    frg = [p.cuda().requires_grad_(True) for p in pool]
    outs = autograd.backbone_stage(model, [[frg[j] for j in idx] for idx in calls_idx])
    fwd = max((o.detach().double() - r).abs().max().item() for o, r in zip(outs, ref_outs))
    assert fwd <= TOL_FP16, fwd
    sum((o * c.cuda()).sum() for o, c in zip(outs, cots)).backward()
    params = dict(model.named_parameters())
    pairs = [(f"frame{j}", frg[j].grad, gfr[j], gfr_emu[j]) for j in range(len(pool))]
    pairs += [(k, params[k].grad, gp[k], gp_emu[k]) for k in gp]
    assert len(pairs) == len(pool) + 2 * (5 * d + 6)
    bad, worst = [], 0.0
    for key, got, ref, emu in pairs:
        assert got is not None, key
        mx = ref.abs().max().item()
        e, e_emu = (got.double() - ref).abs().max().item(), (emu - ref).abs().max().item()
        k_emu = 4.0 if key.endswith("bias") and ".convs." in key and ".convs.3." not in key else 2.0
        worst = max(worst, e / (k_emu * e_emu + 1e-3 * mx))
        if not e <= k_emu * e_emu + 1e-3 * mx:
            bad.append((key, e / mx, e_emu / mx))
    print(f"[light bwd G0={g0} D={d} n={n} ncalls={ncalls} Bc={Bc} {H}x{W}] forward {fwd:.1e}, worst gradient err/bar "
          f"{worst:.3f} over {len(pairs)} tensors")
    assert not bad, bad
    # the "off" channels' ReLU gradient is 0 everywhere: their growth weights and biases get exactly 0
    for i in range(d):
        for c in range(O.C):
            pre = f"RDBs.{i}.convs.{c}.conv.0."
            off = (sd[pre + "bias"] < 0).cuda()
            assert params[pre + "weight"].grad[off].abs().max().item() == 0.0, pre
            assert params[pre + "bias"].grad[off].abs().max().item() == 0.0, pre

    frozen = ("SFENet1.", "RDBs.0.")
    with _deterministic():
        run = lambda **kw: _backbone_grads(model, pool, calls_idx, cots, **kw)
        base = run()
        runs = {"second backward": run(), "recompute": run(mode="recompute"), "frozen": run(frozen=frozen),
                "frozen, no frame gradients": run(frozen=frozen, frame_grad=False)}
    assert all(g is not None for g in base.values())
    for what, grads in runs.items():
        assert list(grads) == list(base), what
        for k, g in grads.items():
            if what.startswith("frozen") and (k.startswith(frozen) or k.startswith("frame") and "no frame" in what):
                assert g is None, (what, k)
            else:
                assert g is not None and torch.equal(_bits(g), _bits(base[k])), (what, k)


def _train_step(net, frames, gts):
    outs = net(*frames)
    loss = sum((o - g).abs().mean() for o, g in zip(outs, gts))
    loss.backward()
    return loss.detach()


def _grads(net):
    return {k: None if p.grad is None else p.grad.clone() for k, p in net.named_parameters()}


@pytest.fixture(scope="module")
def batch():
    fr = [f.cuda() for f in O.synth_frames(6, 2, 64, 64, seed=31, smooth=True)]
    gts = [f.cuda() for f in O.synth_frames(14, 2, 64, 64, seed=32, smooth=True)]
    return fr, gts


@contextlib.contextmanager
def _deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


def test_light_recompute_and_determinism_keep_the_bits(batch):
    """In deterministic mode two steps give the same bits, and activation recomputation gives the default mode's."""
    from bin_b200 import rdn
    fr, gts = batch
    runs = []
    with _deterministic():
        for mode in (None, None, "recompute"):
            net = rdn.set_activation_checkpointing(_light_net().train(), mode)
            loss = _train_step(net, fr, gts)
            runs.append((loss, _grads(net)))
    for loss, grads in runs[1:]:
        assert torch.equal(_bits(loss), _bits(runs[0][0]))
        for k, g in grads.items():
            assert g is not None and torch.equal(_bits(g), _bits(runs[0][1][k])), k


def test_light_frozen_stage_gets_no_gradient(batch):
    from bin_b200 import rdn
    fr, gts = batch
    with _deterministic():
        full = _light_net().train()
        _train_step(full, fr, gts)
        want = _grads(full)
        net = _light_net().train()
        for p in net.model.model1_1.parameters():
            p.requires_grad_(False)
        _train_step(net, fr, gts)
        got = _grads(net)
    for k, g in got.items():
        if k.startswith("model.model1_"):
            assert g is None, k
        else:
            assert g is not None and torch.equal(_bits(g), _bits(want[k])), k


def test_light_guarded_adam_lowers_the_loss(batch):
    from bin_b200.optim import Adam
    fr, gts = batch
    net = _light_net().train()
    opt = Adam(net.parameters(), lr=5e-4, skip_nonfinite=True, max_grad_norm=10.0)
    losses = []
    for _ in range(6):
        opt.zero_grad()
        losses.append(_train_step(net, fr, gts).item())
        opt.step()
    assert all(math.isfinite(v) for v in losses) and opt.skipped_steps == 0
    assert losses[-1] < losses[0], losses
