"""Backward kernels against fp64, held tighter than the whole-network tests can hold them.

Part 1 fuzzes bin_conv_wgrad and the data-gradient convs (bin_conv_fwd over dY with bin_pack_conv_weight_t weights) at
every configuration the backbone backward launches, at every backbone width G0 in {64, 96} and depth D in 1..12, with
the plane offsets it uses (the launch table is backward_layers.py, which test_backward_layers_cpu.py holds to the
library's conv list): segments at non-zero planes, transposed packs with row0 != 0, accumulating and in-place dgrad,
Cout' clipped by store_planes, loss scales 2^-4..2^12, tile remainders, batch 3 and more tiles than SMs.  Every plane of
every input tensor outside the ranges a call is given holds NaN, so a read of a wrong plane shows up as NaN rather than
a small error.

Part 2 runs whole backbones (all four, 1 or 3 calls per launch, batch 1 or 2) on weights whose RDB growth convs keep
every ReLU input at least DELTA away from 0, so fp16 storage cannot flip a ReLU and the gradients can be held to the
fp64 oracle per tensor, with no correlation fallback."""
import math
import random

import pytest
import torch
import torch.nn.functional as F

from backward_layers import spec as _spec
from no_flip import BETA, check_no_relu_near_zero, no_flip_sd, oracle_grads
from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu
NAN = float("nan")


# --------------------------------------------------------------------------------------------------------------------
# part 1: dgrad / wgrad fuzz
# --------------------------------------------------------------------------------------------------------------------
KINDS = ["sfe1", "sfe2", "rdb", "lff", "gff0", "rdb", "up0", "up2", "rdb", "lff", "ring", "rdb"]
NRANDOM = 48
FORCED = {  # name: (kind, forced choices, B, H, W)
    "rdb_1x1": ("rdb", dict(c=3, i=11), 1, 1, 1),
    "rdb_w2": ("rdb", dict(c=2, i=5), 2, 9, 2),
    "rdb_w2_c0": ("rdb", dict(c=0, i=0), 3, 7, 2),
    "rdb_c1_i1_w17": ("rdb", dict(c=1, i=1), 1, 15, 17),
    "lff_h1": ("lff", dict(i=7), 2, 1, 17),
    "lff_i0_w31": ("lff", dict(i=0), 3, 17, 31),
    "sfe1_w1": ("sfe1", dict(cin=60), 3, 15, 1),
    "sfe2_w33": ("sfe2", dict(acc=True), 2, 23, 33),
    "gff0_w47": ("gff0", {}, 1, 9, 47),
    "up0_w15": ("up0", {}, 2, 7, 15),
    "up2_w2": ("up2", {}, 3, 8, 2),
    "ring_w49": ("ring", {}, 2, 25, 49),
    "sfe2_many_tiles": ("sfe2", dict(acc=True), 3, 72, 124),
    "rdb_many_tiles": ("rdb", dict(c=3, i=4), 3, 72, 124),
}
# Every backbone width and depth: each draw picks G0 in {64, 96} and D in 1..12 (and, for an RDB conv or LFF, a quarter
# of the time the recompute layout of the growth maps).  At G0 = 64 the Cout = 64 wgrads run wgrad_kernel<64> (4 taps
# per group) and the G0-row data gradients are 96-row launches clipped to 8 planes; GFF.0's D G0 rows and channels leave
# remainders in the last 96-row block and the last 128-channel wgrad tile.
ARCH_KINDS = ["sfe1", "sfe2", "rdb", "lff", "gff0", "rdb", "up0", "gff1", "rdb", "lff", "gff0", "rdb"]
NARCH = 48
FORCED_ARCH = {  # name: (kind, forced choices incl. g0 and d, B, H, W)
    "g64_sfe1_n2_w1": ("sfe1", dict(g0=64, cin=24), 2, 13, 1),          # 5x5 at N = 64: tap groups 6 x 4 + 1
    "g64_sfe1_n5_w1": ("sfe1", dict(g0=64, cin=60), 3, 15, 1),
    "g64_sfe1_n3_w45": ("sfe1", dict(g0=64, cin=36), 2, 19, 45),        # at W = 1 the last group's tap (kx = 4) reads 0
    "g64_sfe2_w33": ("sfe2", dict(g0=64, acc=True), 2, 23, 33),          # 3x3 at N = 64: tap groups 4 + 4 + 1
    "g64_gff1_many_tiles": ("gff1", dict(g0=64), 3, 72, 124),
    "g64_rdb_c0_i0": ("rdb", dict(g0=64, d=12, c=0, i=0), 2, 9, 21),      # 8 input planes, x = f2, d f2 ends the tensor
    "g64_rdb_c1_i11": ("rdb", dict(g0=64, d=12, c=1, i=11), 1, 17, 30),  # 12 input planes, x = the last-but-one cat block
    "g64_rdb_c2_i5_w2": ("rdb", dict(g0=64, d=12, c=2, i=5), 3, 7, 2),   # 16 input planes
    "g64_rdb_c3_i11": ("rdb", dict(g0=64, d=12, c=3, i=11), 2, 11, 17),  # 20 input planes: a second 128-channel tile
    "g64_rdb_c3_d1": ("rdb", dict(g0=64, d=1, c=3, i=0), 1, 8, 16),
    "g64_rdb_many_tiles": ("rdb", dict(g0=64, d=12, c=3, i=4), 3, 72, 124),
    "g64_lff_i0_d1": ("lff", dict(g0=64, d=1, i=0), 2, 9, 31),           # RDB 0 is also the last: d cat = 8 planes
    "g64_lff_i11_d12": ("lff", dict(g0=64, d=12, i=11), 1, 15, 17),      # dY = the last 8 planes of d cat
    "g64_gff0_d1": ("gff0", dict(g0=64, d=1), 2, 9, 33),                 # 64 rows, 8 planes: half a channel tile
    "g64_gff0_d5": ("gff0", dict(g0=64, d=5), 2, 13, 40),                # 320 rows -> 384, last block stores 4 of 12
    "g64_gff0_d12_many_tiles": ("gff0", dict(g0=64, d=12), 3, 80, 200),
    "g96_gff0_d1": ("gff0", dict(g0=96, d=1), 1, 9, 47),                 # 12 planes: the tile's last box is skipped
    "g96_gff0_d2": ("gff0", dict(g0=96, d=2), 2, 10, 19),                # 24 planes: tiles of 16 + 8
    "g96_gff0_d3": ("gff0", dict(g0=96, d=3), 3, 5, 33),                 # 36 planes: 16 + 16 + 4
    "g64_up0_w15": ("up0", dict(g0=64), 2, 7, 15),                       # 64 channels: 2 of 4 TMA boxes skipped, N = 256
    "g64_rdb_recompute": ("rdb", dict(g0=64, d=12, c=3, i=7, recompute=True), 2, 12, 40),
    "g96_rdb_recompute": ("rdb", dict(g0=96, d=6, c=2, i=3, recompute=True), 1, 16, 35),
    "g64_lff_recompute": ("lff", dict(g0=64, d=6, i=5, recompute=True), 2, 10, 26),
    "g96_lff_recompute": ("lff", dict(g0=96, d=5, i=0, recompute=True), 3, 6, 18),
}


def _case(case):
    if isinstance(case, int):
        rnd = random.Random(case)
        spec = _spec(KINDS[case % len(KINDS)], rnd)
        B, H, W = rnd.choice([1, 2, 3]), rnd.randint(1, 70), rnd.randint(1, 100)
        seed = case
    elif case in FORCED:
        kind, force, B, H, W = FORCED[case]
        rnd = random.Random(case)
        spec = _spec(kind, rnd, **force)
        seed = 1000 + sorted(FORCED).index(case)
    elif case in FORCED_ARCH:
        kind, force, B, H, W = FORCED_ARCH[case]
        rnd = random.Random(case)
        spec = _spec(kind, rnd, **force)
        seed = 3000 + sorted(FORCED_ARCH).index(case)
    else:                                   # "arch<k>"
        k = int(case[4:])
        rnd = random.Random(2000 + k)
        g0, d, recompute = rnd.choice([64, 96]), rnd.randint(1, 12), rnd.random() < 0.25
        spec = _spec(ARCH_KINDS[k % len(ARCH_KINDS)], rnd, g0, d, recompute=recompute)
        B, H, W = rnd.choice([1, 2, 3]), rnd.randint(1, 70), rnd.randint(1, 100)
        seed = 2000 + k
    spec["scale"] = 2.0 ** rnd.randint(-4, 12)
    return spec, B, H, W, seed


def _p8(t, plane0, nplanes, total):
    """NCHW -> fp16 P8 [B, total, H, W, 8] on the GPU: t's channels fill planes [plane0, plane0 + nplanes) (channels past
    t's count are zero, as the backbone writes them); every other plane is NaN."""
    B, Cc, H, W = t.shape
    assert Cc <= 8 * nplanes and plane0 + nplanes <= total
    out = torch.full((B, total, H, W, 8), NAN, dtype=torch.float16)
    blk = torch.zeros((B, 8 * nplanes, H, W))
    blk[:, :Cc] = t
    out[:, plane0:plane0 + nplanes] = blk.view(B, nplanes, 8, H, W).permute(0, 1, 3, 4, 2).half()
    return out.cuda()


def _planes_nchw(p, plane0, nplanes):
    """P8 planes [plane0, plane0 + nplanes) -> fp64 NCHW on the CPU (all 8 nplanes channels)."""
    B, _, H, W, _ = p.shape
    return p[:, plane0:plane0 + nplanes].permute(0, 1, 4, 2, 3).reshape(B, 8 * nplanes, H, W).double().cpu()


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


def _tiles_over_sms(B, H, W, k):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    conv_tw = 32 - 2 * (k // 2)                       # output columns of a conv tile (internal.h kTWH - 2 pad) x 8 rows
    return B * -(-H // 8) * -(-W // 16) > sms, B * -(-H // 8) * -(-W // conv_tw) > sms


@pytest.mark.parametrize("case", list(range(NRANDOM)) + sorted(FORCED) + [f"arch{k}" for k in range(NARCH)] + sorted(FORCED_ARCH))
def test_backward_conv_fuzz(case):
    from bin_b200 import ops
    from bin_b200._lib import Act, check, lib
    spec, B, H, W, seed = _case(case)
    cin, cout, k, scale = spec["cin"], spec["cout"], spec["k"], spec["scale"]
    where = (case, spec.get("tag", ""), cin, cout, k, B, H, W, scale)
    if isinstance(case, str) and case.endswith("many_tiles"):
        assert all(_tiles_over_sms(B, H, W, k)), where
    g = torch.Generator().manual_seed(7000 + seed)
    x = torch.randn((B, cin, H, W), generator=g).half().float()
    w = (torch.randn((cout, cin, k, k), generator=g) / math.sqrt(cin * k * k)).half().float()
    dy = torch.randn((B, cout, H, W), generator=g).half().float()     # the stored (loss-scaled) gradient
    # fp64 CPU reference on the same fp16-rounded operands
    x64, w64 = x.double().requires_grad_(True), w.double().requires_grad_(True)
    gx_ref, gw_ref = torch.autograd.grad((F.conv2d(x64, w64, padding=k // 2) * dy.double()).sum(), [x64, w64])
    gw_ref = gw_ref / scale
    st = torch.cuda.current_stream().cuda_stream

    # ---- wgrad: dw += (1/scale) X^T dY, segments at the backbone's plane offsets
    segs, c0 = [], 0
    for total, plane0, np_ in spec["x"]:
        c1 = min(c0 + 8 * np_, cin)
        segs.append((_p8(x[:, c0:c1], plane0, np_, total), plane0, np_))
        c0 += 8 * np_
    assert c0 >= cin
    dy_total, dy_plane0 = spec["dy"]
    dy_np = (cout + 31) // 32 * 4
    dyt = _p8(dy, dy_plane0, dy_np, dy_total)
    inputs = [s[0] for s in segs] + [dyt]
    before = [t.clone() for t in inputs]
    x1 = segs[1] if len(segs) > 1 else (None, 0, 0)
    a1 = ops.act_view(x1[0]) if x1[0] is not None else Act(None, 0, 0, 0, 0)
    sc = torch.full((1,), scale, device="cuda")
    wsp = torch.empty(lib().bin_conv_wgrad_workspace_bytes(), dtype=torch.uint8, device="cuda")
    ref_max = gw_ref.abs().max().item()
    dw0 = torch.randn(w.shape, generator=g).cuda() * ref_max             # wgrad adds into a dw that is not zero
    runs = []
    for _ in range(2):
        dw = dw0.clone()
        check(lib().bin_conv_wgrad(ops.act_view(segs[0][0]), segs[0][1], segs[0][2], a1, x1[1], x1[2], ops.act_view(dyt),
                                   dy_plane0, cout, cin, k, sc.data_ptr(), dw.data_ptr(), wsp.data_ptr(), st))
        runs.append(dw)
    torch.cuda.synchronize()
    err = ((runs[0].double() - dw0.double()).cpu() - gw_ref).abs().max().item()
    ratios = {"wgrad": err / (1e-4 * ref_max)}
    assert err <= 1e-4 * ref_max, ("wgrad", where, err, ref_max)
    assert _same_bits(runs[0], runs[1]), ("wgrad is not bit-reproducible", where)       # fixed-order slab reduction
    for t, t0 in zip(inputs, before):
        assert _same_bits(t, t0), ("wgrad wrote into an input", where)

    # ---- dgrad: dX (+)= conv(dY, V) through the transposed pack, clipped to store_planes
    cin_pad_t = (cout + 31) // 32 * 32
    wc = w.cuda()
    for d in spec["dgrad"]:
        row0, nrows, acc = d["row0"], d["nrows"], d["acc"]
        out_total, out_plane0, nstore = d["out"]
        cout_pad_t = (nrows + 95) // 96 * 96
        wt = torch.empty(cout_pad_t * cin_pad_t * k * k, dtype=torch.float16, device="cuda")
        check(lib().bin_pack_conv_weight_t(wc.data_ptr(), cout, cin, k, row0, nrows, cout_pad_t, cin_pad_t,
                                           wt.data_ptr(), st))
        prefill = (torch.randn((B, nstore, H, W, 8), generator=g) * gx_ref.std().item()).half().cuda()
        if out_total is None:               # in place: the output planes are a range of the dY tensor itself
            outt = _p8(dy, dy_plane0, dy_np, dy_total)
        else:
            outt = torch.randn((B, out_total, H, W, 8), generator=g).half().cuda()
        outt[:, out_plane0:out_plane0 + nstore] = prefill
        out0 = outt.clone()
        zero_bias = torch.zeros(cout_pad_t, device="cuda")
        ops.conv_fwd(outt if out_total is None else dyt, wt, zero_bias, k, cout_pad_t, in0_plane0=dy_plane0,
                     in0_planes=dy_np, out=outt, out_plane0=out_plane0, res=outt if acc else None, res_plane0=out_plane0,
                     store_planes=nstore)
        torch.cuda.synchronize()
        exp = torch.zeros((B, 8 * nstore, H, W), dtype=torch.float64)
        exp[:, :nrows] = gx_ref[:, row0:row0 + nrows]
        if acc:
            exp += _planes_nchw(prefill, 0, nstore)
        got = _planes_nchw(outt, out_plane0, nstore)
        err = (got - exp).abs().max().item()
        ratios[f"dgrad rows {row0}+{nrows}"] = err / (2e-3 * exp.abs().max().item())
        assert err <= 2e-3 * exp.abs().max().item(), ("dgrad", row0, nrows, acc, where, err, exp.abs().max().item())
        keep = torch.ones(outt.shape[1], dtype=torch.bool)
        keep[out_plane0:out_plane0 + nstore] = False
        assert _same_bits(outt[:, keep], out0[:, keep]), ("dgrad wrote outside its planes", row0, nrows, where)
        if out_total is not None:
            assert _same_bits(dyt, before[-1]), ("dgrad wrote into dY", where)
    print(f"[bwd fuzz] {case} {spec.get('tag', '')} {cin}->{cout} k={k} B={B} {H}x{W}: worst err/bar "
          + ", ".join(f"{key} {r:.3f}" for key, r in ratios.items()))


# --------------------------------------------------------------------------------------------------------------------
# part 2: whole backbones with no ReLU input near 0
# --------------------------------------------------------------------------------------------------------------------
BACKBONES = [("model1_1", 2, 201), ("model2_1", 3, 202), ("model3_1", 5, 203), ("model4_1", 5, 204)]
LAUNCHES = [(1, 1, 30, 50), (1, 2, 44, 68), (3, 1, 44, 68), (3, 2, 30, 50)]     # (ncalls, Bc, full-res H, W)


@pytest.mark.parametrize("ncalls,Bc,H,W", LAUNCHES)
@pytest.mark.parametrize("name,n,seed", BACKBONES)
def test_backbone_backward_without_relu_flips(name, n, seed, ncalls, Bc, H, W):
    from bin_b200 import autograd, rdn
    cls = {2: rdn.RDN_residual_interp_2_input, 3: rdn.RDN_residual_interp_2_1_input, 5: rdn.RDN_residual_interp_4_1_input}[n]
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        # call k reads pool frames k .. k+n-2 and k+1 again: one frame tensor feeds two calls and, for n >= 3, two slots
        # of one call (as pyramid_apply does), so autograd has to sum the contributions
        pool = O.synth_frames(ncalls + max(n - 2, 1), Bc, H, W, seed=seed + 17 * ncalls + Bc)
        calls_idx = [list(range(k, k + n - 1)) + [k + 1] for k in range(ncalls)]
        cots = [c - 0.5 for c in O.synth_frames(ncalls, Bc, H, W, seed=seed + 1)]
        pool64 = [p.to("cuda", torch.float64) for p in pool]
        sd = {k: v.cpu() for k, v in no_flip_sd(n, seed, [[pool64[j] for j in idx] for idx in calls_idx]).items()}
        margin, cv = check_no_relu_near_zero([[pool64[j] for j in idx] for idx in calls_idx], sd)
        ref_outs, gfr, gp = oracle_grads(pool, calls_idx, cots, sd, emulate=False)
        _, gfr_emu, gp_emu = oracle_grads(pool, calls_idx, cots, sd, emulate=True)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32

    model = cls(G0=96, D=12)
    model.load_state_dict(sd, strict=True)
    model = model.cuda()
    frg = [p.cuda().requires_grad_(True) for p in pool]
    outs = autograd.backbone_stage(model, [[frg[j] for j in idx] for idx in calls_idx])
    fwd = max((o.detach().double() - r).abs().max().item() for o, r in zip(outs, ref_outs))
    assert fwd <= 1e-3, fwd
    sum((o * c.cuda()).sum() for o, c in zip(outs, cots)).backward()

    params = dict(model.named_parameters())
    rows, bad = [], []
    pairs = [(f"frame{j}", frg[j].grad, gfr[j], gfr_emu[j]) for j in range(len(pool))]
    pairs += [(k, params[k].grad, gp[k], gp_emu[k]) for k in gp]
    assert len(pairs) == len(pool) + 132
    for key, got, ref, emu in pairs:
        assert got is not None, key
        m = ref.abs().max().item()
        e, e_emu = (got.double() - ref).abs().max().item(), (emu - ref).abs().max().item()
        rows.append((e / m, e_emu / m, key))
        # the dY of growth conv c < 3 is summed in fp16, in place, over 4 - c launches (LFF, then convs c+1..3), where the
        # oracle rounds the finished sum once; the bias gradient (a plain sum of that dY over all pixels) shows it most
        k_emu = 4.0 if key.endswith("bias") and ".convs." in key and ".convs.3." not in key else 2.0
        if not e <= k_emu * e_emu + 1e-3 * m:
            bad.append((key, e / m, e_emu / m))
    # the "off" channels' ReLU gradient is 0 everywhere: their growth weights and biases get exactly 0
    for i in range(O.D):
        for c in range(O.C):
            pre = f"RDBs.{i}.convs.{c}.conv.0."
            off = (sd[pre + "bias"] < 0).cuda()
            assert params[pre + "weight"].grad[off].abs().max().item() == 0.0, pre
            assert params[pre + "bias"].grad[off].abs().max().item() == 0.0, pre
    cu, em = sorted(r[0] for r in rows), sorted(r[1] for r in rows)
    print(f"[bwd no-flip {name} ncalls={ncalls} Bc={Bc} {H}x{W}] per-tensor max error / tensor max over {len(rows)} tensors: "
          f"CUDA vs fp64 worst {cu[-1]:.2e} median {cu[len(cu) // 2]:.2e} | fp16-storage oracle vs fp64 worst {em[-1]:.2e} "
          f"median {em[len(em) // 2]:.2e} | forward {fwd:.1e} | ReLU margin {margin / BETA:.3f} BETA, min std/mean {cv:.3f}")
    assert not bad, sorted(bad, key=lambda r: -r[1])[:8]
