"""Forward kernels against fp64, per element, with bars derived from the arithmetic instead of fitted to a run.

Part 1 fuzzes bin_conv_fwd over all 14 kernel instantiations (P8 <32,3,SX> <96,3> <96,5> <96,1> and PIXSHUF <128,3> and
FINAL <16,3,SX> in both precisions; P8 <32,3,plain> and FINAL <16,3,plain> in fp16), at the segment and plane layouts
the backbone launches (RDB conv c of RDB i reading cat[12(i-1), +12) and g[g0, +4c), the LFF writing planes 12i of the
tensor it reads at 12(i-1), ...), with store_planes, cout_pad 192, sub-ranges of all three epilogues, FINAL call tables,
tile remainders, more tiles than SMs, both weight paths (resident in shared memory or streamed per stage) and three
activation magnitudes.  Every plane of every tensor outside a call's ranges holds NaN, every output element the call must
not write holds a sentinel, and both keep their bits.  The first 36 cases are the draws of the earlier conv fuzz.
Part 2 holds bin_rdb_tail_fwd to fp64 at the backbone's plane offsets, part 3 bin_pack_frames(_p) bit for bit to a torch
restatement, part 4 bin_convlstm_fwd to fp64 with 1, 2 and 3 cells per launch, each cell of a group bit for bit to its
own one-cell launch.

Bars (u = 2^-24, the fp32 unit roundoff; A = sum |x||w| + |b| + |res| of the element, an fp64 conv of absolute values):
  fp16 P8 / PIXSHUF   |got - ref| <= ulp16(ref) + C_F16 u A          ref: fp64 on the same fp16 operands
  FINAL (fp16)        |got - ref| <= ulp32(ref) + C_FINAL u A + (n+1) u sum_f |frame_f|
  X3 (fp32-accurate)  ref: fp64 on the ORIGINAL fp32 operands.  Each operand pair hi + lo is within 2^-22 |v| of v, or
                      2^-25 absolute where lo is an fp16 subnormal (|v| < ~2^-3; weights are split as 2^8 w, so 2^-33 on
                      w); the dropped lo*lo term is below 2^-22 |x w|; the output split adds 2^-22 |out| + 2^-25:
                      |got - ref| <= C_X3 u (A + |res|) + 2^-22 (3 A + |ref| + 2 |res|) + 2^-25 (W1 + 2) + 2^-33 X1
                      (W1 = sum |w| of the output channel, X1 = sum |x| of the receptive field), with the FINAL terms
                      above in place of the output split for the final epilogue.
  RDB tail            the fp16 bar, plus sum_j |w_lff[:, g3_j]| (ulp16(g3_j) + C_TAIL u A3_j): the kernel rounds its own
                      fp32 g3 to fp16, which can land one ulp away from the rounded fp64 g3.
  ConvLSTM            gate sums: K_LSTM u G (54 or 27 FMAs, the bias and the forget bias); sigmoid / tanh add T_LSTM
                      (the kernel's documented bound) and carry the gate error with slope 1/4 and 1; c and h follow by
                      the product rule, the c term scaled by |c_prev|.
  pack                torch.equal.
"""
import math
import random
import statistics

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
NAN = float("nan")
SENTINEL = -1234.0              # exact in fp16: hi = -1234, lo = 0
U = 2.0 ** -24
C_F16 = 32.0
C_FINAL = 32.0
C_X3 = 32.0
C_TAIL = 32.0
K_LSTM = 56.0
T_LSTM = 3e-7
DEV = "cuda"
RATIOS = {}                     # (label, precision) -> [worst error / bar of each case]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(RATIOS):
        r = sorted(RATIOS[key])
        print(f"[fwd fuzz] {key[0]:<22} {key[1]:<4} cases {len(r):3d}  worst err/bar {r[-1]:.3f}  median {statistics.median(r):.3f}")


def _record(label, prec, ratio):
    RATIOS.setdefault((label, prec), []).append(ratio)


def ulp16(v):
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def ulp32(v):
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 23)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


def _x3_plane(lp):
    return 2 * (lp & ~3) + (lp & 3)


# --------------------------------------------------------------------------------------------------------------------
# kernel selection, as launch_conv_t / launch_inst pick it (internal.h, conv_igemm.cu)
# --------------------------------------------------------------------------------------------------------------------
SMEM_MAX, CTRL, MAX_RESIDENT = 227 * 1024, 2048, 8


def _inst(spec):
    """(label, NT, KS, SX) of the kernel bin_conv_fwd runs for this spec."""
    k, cp, epi, var = spec["k"], spec["cout_pad"], spec["epi"], spec["variant"]
    if epi == 1:
        return "pixshuf<128,3>", 128, 3, False
    if epi == 2:
        return ("final<16,3,SX>" if var == 0 else "final<16,3,plain>"), 16, 3, var == 0
    if k == 3 and cp == 32:
        return ("p8<32,3,SX>" if var == 0 else "p8<32,3,plain>"), 32, 3, var == 0
    return f"p8<96,{k}>", 96, k, False


def _resident(spec, x3):
    """launch_inst: weights stay in shared memory iff nh == 1, <= 8 chunks, and >= 3 activation stages still fit."""
    _, nt, ks, sx = _inst(spec)
    nh = spec["cout_pad"] // nt
    nchunks = (3 if x3 else 1) * sum(s[2] // 4 for s in spec["segs"])
    rows = 8 if ks == 5 else 8 + 2 * (ks // 2)
    a_bytes = 4 * rows * 32 * 16
    nmma = nt * ks if sx else nt
    w_chunk = (ks if sx else ks * ks) * 4 * nmma * 16
    xs = 96 * nt if sx else 0
    return nh == 1 and nchunks <= MAX_RESIDENT and CTRL + nchunks * w_chunk + xs + 3 * a_bytes + 256 <= SMEM_MAX


def _ntiles(spec, B, H, W, sub):
    _, nt, ks, _ = _inst(spec)
    b0, nb, y0, ny = sub if sub else (0, B, 0, H)
    return nb * -(-ny // 8) * -(-W // (32 - 2 * (ks // 2))) * (spec["cout_pad"] // nt)


# --------------------------------------------------------------------------------------------------------------------
# part 1: the conv specs
# --------------------------------------------------------------------------------------------------------------------
def _spec(kind, rnd, **force):
    """One conv launch.  segs: input segments (tensor, plane0, planes); out / res: (tensor, plane0); tensors: name ->
    (logical planes, spatial factor).  cin: channels with data (the rest of the segment planes hold zeros, as the packer
    writes them for SFENet1)."""
    pick = lambda key, choices: force[key] if key in force else rnd.choice(choices)
    base = dict(variant=0, epi=0, relu=False, res=None, store=0, final=None)
    if kind == "sfe1":                       # SFENet1 5x5 on the packed frames: 24/36/60 channels in 4 or 8 planes
        cin = pick("cin", [24, 36, 60])
        xp = (cin + 31) // 32 * 4
        return dict(base, k=5, cin=cin, cout=96, cout_pad=96, tensors=dict(x0=(xp, 1), f1=(12, 1)), segs=[("x0", 0, xp)],
                    out=("f1", 0), tag=f"cin={cin}")
    if kind == "sfe2":
        return dict(base, k=3, cin=96, cout=96, cout_pad=96, tensors=dict(f1=(12, 1), f2=(12, 1)), segs=[("f1", 0, 12)],
                    out=("f2", 0))
    if kind == "gff1":                       # GFF.1 with the residual f1
        return dict(base, k=3, cin=96, cout=96, cout_pad=96, tensors=dict(t1=(12, 1), t2=(12, 1), f1=(12, 1)),
                    segs=[("t1", 0, 12)], out=("t2", 0), res=("f1", 0))
    if kind == "rdb":                        # conv c of RDB i: cat[12(i-1), +12) or f2, then g[g0, +4c) -> g[g0 + 4c, +4)
        c, i = pick("c", range(4)), pick("i", range(12))
        train = pick("train", [False, True])
        g0 = 16 * i if train else 0
        tensors = dict(g=(192 if train else 16, 1))
        if i:
            tensors["cat"] = (144, 1)
            segs = [("cat", 12 * (i - 1), 12)]
        else:
            tensors["f2"] = (12, 1)
            segs = [("f2", 0, 12)]
        if c:
            segs.append(("g", g0, 4 * c))
        return dict(base, k=3, cin=96 + 32 * c, cout=32, cout_pad=32, variant=pick("variant", [0, 0, 1]), relu=True,
                    tensors=tensors, segs=segs, out=("g", g0 + 4 * c), tag=f"c={c} i={i} g0={g0}")
    if kind == "lff":                        # LFF of RDB i: residual cat[12(i-1)], output cat[12 i] of the same tensor
        i = pick("i", range(12))
        train = pick("train", [False, True])
        g0 = 16 * i if train else 0
        tensors = dict(g=(192 if train else 16, 1), cat=(144, 1))
        if i:
            xin = ("cat", 12 * (i - 1), 12)
        else:
            tensors["f2"] = (12, 1)
            xin = ("f2", 0, 12)
        return dict(base, k=1, cin=224, cout=96, cout_pad=96, tensors=tensors, segs=[xin, ("g", g0, 16)],
                    out=("cat", 12 * i), res=xin[:2], tag=f"i={i} g0={g0}")
    if kind == "gff0":
        return dict(base, k=1, cin=1152, cout=96, cout_pad=96, tensors=dict(cat=(144, 1), t1=(12, 1)),
                    segs=[("cat", 0, 144)], out=("t1", 0))
    if kind == "up0":                        # UPNet.0 + PixelShuffle(2)
        op0 = pick("op0", [0, 0, 4])
        return dict(base, k=3, cin=96, cout=256, cout_pad=256, epi=1, tensors=dict(t2=(12, 1), u=(8 + op0, 2)),
                    segs=[("t2", 0, 12)], out=("u", op0), tag=f"op0={op0}")
    if kind == "up2":                        # UPNet.2 + mean(frames) -> fp32 NCHW per call
        cin = pick("cin", [64])
        return dict(base, k=3, cin=cin, cout=3, cout_pad=16, epi=2, variant=pick("variant", [0, 0, 1]),
                    tensors=dict(u=(cin // 8, 1)), segs=[("u", 0, cin // 8)], out=None,
                    final=dict(ncalls=pick("ncalls", [1, 2, 3]), nframes=pick("nframes", [2, 3, 5]),
                               shared=pick("shared", [False, True])))
    if kind == "wide":                       # cout_pad 192 (nh = 2) for the 96-wide kernels, optionally clipped
        k = pick("k", [3, 1])
        cout = pick("cout", [150, 192])
        store = pick("store", [0, 0, 17, 24])
        res = pick("res", [False, True])
        return dict(base, k=k, cin=96, cout=cout, cout_pad=192, tensors=dict(a=(16, 1), o=(28, 1), r=(32, 1)),
                    segs=[("a", 4, 12)], out=("o", 4), res=("r", 4) if res else None, store=store,
                    tag=f"k={k} cout={cout} store={store} res={res}")
    if kind == "store":                      # store_planes below cout_pad / 8 on the 96-wide kernels
        k = pick("k", [3, 1, 5])
        store = pick("store", [1, 4, 5, 11])
        return dict(base, k=k, cin=64 if k == 5 else 96, cout=96, cout_pad=96, tensors=dict(a=(16, 1), o=(20, 1)),
                    segs=[("a", 4, 8 if k == 5 else 12)], out=("o", 8), store=store, relu=pick("relu", [False, True]),
                    tag=f"k={k} store={store}")
    if kind == "generic":                    # any instantiation with chosen chunk counts (resident / streamed weights)
        inst, cin = force["inst"], force["cin"]
        k, cp, epi, var = dict(sx=(3, 32, 0, 0), plain=(3, 32, 0, 1), p3=(3, 96, 0, 0), p5=(5, 96, 0, 0), p1=(1, 96, 0, 0),
                               ps=(3, 256, 1, 0), fsx=(3, 16, 2, 0), fplain=(3, 16, 2, 1))[inst]
        planes = cin // 8
        out = None if epi == 2 else ("o", 0)
        tensors = dict(a=(planes, 1))
        if epi == 0:
            tensors["o"] = (cp // 8, 1)
        elif epi == 1:
            tensors["o"] = (8, 2)
        return dict(base, k=k, cin=cin, cout=3 if epi == 2 else cp, cout_pad=cp, epi=epi, variant=var, relu=epi == 0,
                    tensors=tensors, segs=[("a", 0, planes)], out=out,
                    final=dict(ncalls=1, nframes=2, shared=False) if epi == 2 else None, tag=f"{inst} cin={cin}")
    raise ValueError(kind)


# the layers of the earlier conv fuzz (all at plane 0), kept as they were drawn
OLD_LAYERS = [  # (cin, cout, k, epilogue, relu, residual, split)
    (24, 96, 5, 0, False, False, None), (36, 96, 5, 0, False, False, None), (60, 96, 5, 0, False, False, None),
    (96, 96, 3, 0, False, True, None), (96, 32, 3, 0, True, False, None), (128, 32, 3, 0, True, False, 96),
    (160, 32, 3, 0, True, False, 96), (192, 32, 3, 0, True, False, 96), (224, 96, 1, 0, False, True, 96),
    (1152, 96, 1, 0, False, False, None), (96, 256, 3, 1, False, False, None), (64, 3, 3, 2, False, False, None),
]
NOLD = 36


def _old_case(seed):
    rnd = random.Random(seed)
    cin, cout, k, epi, relu, res, split = OLD_LAYERS[seed % len(OLD_LAYERS)]
    B = rnd.choice([1, 2, 3])
    H, W = rnd.randint(1, 70), rnd.randint(1, 100)
    sub = None
    if epi == 0 and rnd.random() < 0.4:
        b0 = rnd.randrange(B)
        y0 = rnd.randrange(H)
        sub = (b0, rnd.randint(1, B - b0), y0, rnd.randint(1, H - y0))
    cin_pad = (cin + 31) // 32 * 32
    cout_pad = 16 if cout == 3 else cout
    p = cin_pad // 8
    segs = [("a", 0, p)] if split is None else [("a", 0, split // 8), ("b", 0, p - split // 8)]
    tensors = {s[0]: (s[2], 1) for s in segs}
    out = None
    if epi == 0:
        tensors["o"] = (cout_pad // 8, 1)
        out = ("o", 0)
    elif epi == 1:
        tensors["o"] = (8, 2)
        out = ("o", 0)
    if res:
        tensors["r"] = (cout_pad // 8, 1)
    spec = dict(k=k, cin=cin, cout=cout, cout_pad=cout_pad, variant=0, epi=epi, relu=relu, tensors=tensors, segs=segs,
                out=out, res=("r", 0) if res else None, store=0, tag="earlier fuzz",
                final=dict(ncalls=B, nframes=2 + seed % 4, shared=False) if epi == 2 else None)
    if epi == 2:
        spec["final"]["Bc"] = 1
    return spec, B, H, W, sub, False, 1.0


KINDS = ["sfe1", "sfe2", "gff1", "rdb", "lff", "gff0", "up0", "up2", "rdb", "lff", "wide", "store", "rdb", "up2"]
NRANDOM = 64
MAGS = {"f16": [1.0, 2.0 ** -12, 2.0 ** 5], "x3": [1.0, 2.0 ** -12, 2.0 ** 5, 2.0 ** -5]}


def _dim(rnd, mults):
    m = rnd.choice(mults)
    return max(1, rnd.choice([1, 2, m * rnd.randint(1, 3) + rnd.choice([-1, 0, 1]), rnd.randint(1, 100)]))


def _random_case(seed):
    rnd = random.Random(10_000 + seed)
    spec = _spec(KINDS[seed % len(KINDS)], rnd)
    plain = spec["variant"] == 1
    x3 = (not plain) and rnd.random() < 0.4
    B = rnd.choice([1, 2, 3])
    H, W = _dim(rnd, [8]), _dim(rnd, [30, 28, 32])
    if spec["epi"] == 2:
        fin = spec["final"]
        fin["Bc"] = rnd.choice([1, 2, 3])
        B = fin["ncalls"] * fin["Bc"]
    sub = None
    if rnd.random() < 0.4:
        b0 = rnd.randrange(B)
        y0 = rnd.randrange(H)
        sub = (b0, rnd.randint(1, B - b0), y0, rnd.randint(1, H - y0))
    return spec, B, H, W, sub, x3, rnd.choice(MAGS["x3" if x3 else "f16"])


MANY = (3, 72, 130)               # more conv tiles than SMs for every kernel (8-row tiles, 28..32 columns)
FORCED = {  # name: (kind, forced choices, B, H, W, sub, x3, magnitude)
    # the backbone's own layouts at their plane offsets
    "rdb_c3_i11_train": ("rdb", dict(c=3, i=11, train=True, variant=0), 2, 17, 61, None, False, 1.0),
    "rdb_c2_i5_x3": ("rdb", dict(c=2, i=5, train=False, variant=0), 1, 9, 31, None, True, 1.0),
    "rdb_c1_i1_plain": ("rdb", dict(c=1, i=1, train=True, variant=1), 3, 8, 30, (1, 2, 3, 4), False, 1.0),
    "rdb_c0_i0_x3_sub": ("rdb", dict(c=0, i=0, train=False, variant=0), 3, 15, 29, (2, 1, 5, 9), True, 2.0 ** -5),
    "lff_i7_train": ("lff", dict(i=7, train=True), 2, 16, 33, None, False, 1.0),
    "lff_i11_x3": ("lff", dict(i=11, train=True), 1, 7, 32, (0, 1, 2, 3), True, 1.0),
    "lff_i0_x3": ("lff", dict(i=0, train=False), 2, 9, 31, None, True, 2.0 ** -12),
    "sfe1_24_x3": ("sfe1", dict(cin=24), 2, 9, 27, None, True, 1.0),
    "sfe1_60_sub": ("sfe1", dict(cin=60), 3, 17, 57, (1, 1, 4, 9), False, 2.0 ** 5),
    "gff1_x3_sub": ("gff1", {}, 3, 16, 61, (0, 2, 7, 8), True, 1.0),
    "gff0_w1": ("gff0", {}, 2, 7, 1, None, False, 1.0),
    "gff0_x3": ("gff0", {}, 1, 8, 33, None, True, 1.0),
    "up0_op4_sub": ("up0", dict(op0=4), 3, 10, 31, (1, 2, 3, 5), False, 1.0),
    "up0_x3_sub": ("up0", dict(op0=4), 2, 9, 29, (0, 1, 8, 1), True, 2.0 ** -12),
    "wide_k3_store17_res": ("wide", dict(k=3, cout=150, store=17, res=True), 2, 9, 31, None, False, 1.0),
    "wide_k1_x3_res": ("wide", dict(k=1, cout=192, store=24, res=True), 2, 9, 33, (1, 1, 0, 9), True, 1.0),
    "wide_k3_x3": ("wide", dict(k=3, cout=192, store=0, res=False), 1, 16, 30, None, True, 2.0 ** 5),
    "store1_k5": ("store", dict(k=5, store=1, relu=False), 2, 8, 28, None, False, 1.0),
    "store5_k3_x3": ("store", dict(k=3, store=5, relu=True), 2, 9, 31, None, True, 1.0),
    "store11_k1_x3": ("store", dict(k=1, store=11, relu=False), 1, 9, 65, (0, 1, 1, 7), True, 2.0 ** -12),
    # FINAL tables: ncalls 1..6, Bc 1..3, nframes 2/3/5, a frame shared by two calls, sub-ranges
    "final_6x1_n2_shared": ("up2", dict(ncalls=6, nframes=2, shared=True, variant=0), 6, 9, 31, None, False, 1.0),
    "final_1x3_n5": ("up2", dict(ncalls=1, nframes=5, shared=False, variant=0), 3, 16, 29, None, True, 1.0),
    "final_2x3_n3_sub": ("up2", dict(ncalls=2, nframes=3, shared=True, variant=0), 6, 17, 33, (2, 3, 5, 9), False, 1.0),
    "final_3x2_n5_x3_sub": ("up2", dict(ncalls=3, nframes=5, shared=True, variant=0), 6, 8, 30, (1, 4, 0, 3), True, 2.0 ** -5),
    "final_4x1_n3_plain": ("up2", dict(ncalls=4, nframes=3, shared=True, variant=1), 4, 7, 61, (1, 2, 2, 4), False, 2.0 ** 5),
    "final_5x1_n2_x3": ("up2", dict(ncalls=5, nframes=2, shared=False, variant=0), 5, 2, 2, None, True, 1.0),
    # H or W of 1 and 2
    "sfe2_1x1": ("sfe2", {}, 3, 1, 1, None, False, 1.0),
    "rdb_h1_x3": ("rdb", dict(c=3, i=2, train=False, variant=0), 2, 1, 45, None, True, 1.0),
    "rdb_w2_plain": ("rdb", dict(c=2, i=3, train=True, variant=1), 2, 9, 2, None, False, 1.0),
    "up0_h2_w1": ("up0", dict(op0=0), 2, 2, 1, None, False, 1.0),
    "final_w1": ("up2", dict(ncalls=2, nframes=3, shared=True, variant=0), 2, 5, 1, None, False, 1.0),
    # resident / streamed weights where the host's rule allows both
    "res_sx_x3": ("generic", dict(inst="sx", cin=64), 2, 9, 31, None, True, 1.0),
    "stream_sx": ("generic", dict(inst="sx", cin=288), 2, 9, 31, None, False, 1.0),
    "stream_plain": ("generic", dict(inst="plain", cin=288), 2, 9, 31, None, False, 1.0),
    "res_p3_x3": ("generic", dict(inst="p3", cin=32), 2, 9, 31, None, True, 1.0),
    "res_p5": ("generic", dict(inst="p5", cin=32), 2, 9, 29, None, False, 1.0),
    "res_p1_x3": ("generic", dict(inst="p1", cin=64), 2, 9, 33, None, True, 1.0),
    "stream_fsx": ("generic", dict(inst="fsx", cin=288), 1, 9, 31, None, False, 1.0),
    "stream_fsx_x3": ("generic", dict(inst="fsx", cin=96), 1, 9, 31, None, True, 1.0),
    "stream_fplain": ("generic", dict(inst="fplain", cin=288), 1, 9, 31, None, False, 1.0),
    # more tiles than SMs, every instantiation and precision
    "many_sx": ("rdb", dict(c=3, i=4, train=True, variant=0), *MANY, None, False, 1.0),
    "many_sx_x3": ("rdb", dict(c=1, i=4, train=False, variant=0), *MANY, None, True, 1.0),
    "many_plain": ("rdb", dict(c=2, i=9, train=True, variant=1), *MANY, None, False, 1.0),
    "many_p3": ("gff1", {}, *MANY, None, False, 1.0),
    "many_p3_x3": ("sfe2", {}, *MANY, None, True, 1.0),
    "many_p5": ("sfe1", dict(cin=36), *MANY, None, False, 1.0),
    "many_p5_x3": ("sfe1", dict(cin=60), *MANY, None, True, 1.0),
    "many_p1": ("lff", dict(i=3, train=True), *MANY, None, False, 1.0),
    "many_p1_x3": ("lff", dict(i=6, train=False), *MANY, None, True, 1.0),
    "many_pixshuf": ("up0", dict(op0=0), *MANY, None, False, 1.0),
    "many_pixshuf_x3": ("up0", dict(op0=4), *MANY, None, True, 1.0),
    "many_final": ("up2", dict(ncalls=3, nframes=2, shared=True, variant=0), *MANY, None, False, 1.0),
    "many_final_x3": ("up2", dict(ncalls=1, nframes=3, shared=False, variant=0), *MANY, None, True, 1.0),
    "many_final_plain": ("up2", dict(ncalls=3, nframes=5, shared=True, variant=1), *MANY, None, False, 1.0),
}


def _forced_case(name):
    kind, force, B, H, W, sub, x3, mag = FORCED[name]
    spec = _spec(kind, random.Random(name), **force)
    if spec["epi"] == 2:
        spec["final"]["Bc"] = B // spec["final"]["ncalls"]
        assert spec["final"]["Bc"] * spec["final"]["ncalls"] == B, name
    return spec, B, H, W, sub, x3, mag


def _to_device(vals, x3):
    """Logical fp64 values (B, 8 planes, Hs, Ws) -> P8 fp16 [B, planes, Hs, Ws, 8], or its (hi, lo) layout for x3."""
    B, C8, Hs, Ws = vals.shape
    p8 = vals.view(B, C8 // 8, 8, Hs, Ws).permute(0, 1, 3, 4, 2).float()
    if not x3:
        return p8.half().contiguous()
    hi = p8.half()
    lo = (p8 - hi.float()).half()
    planes = C8 // 8
    out = torch.empty((B, 2 * planes, Hs, Ws, 8), dtype=torch.float16, device=vals.device)
    for lp in range(planes):
        out[:, _x3_plane(lp)] = hi[:, lp]
        out[:, _x3_plane(lp) + 4] = lo[:, lp]
    return out


def _from_device(t, plane0, nplanes, x3):
    """Logical planes [plane0, +nplanes) -> fp64 NCHW (hi + lo for x3)."""
    if x3:
        idx = torch.tensor([_x3_plane(lp) for lp in range(plane0, plane0 + nplanes)], device=t.device)
        v = t[:, idx].double() + t[:, idx + 4].double()
    else:
        v = t[:, plane0:plane0 + nplanes].double()
    B, _, Hs, Ws, _ = v.shape
    return v.permute(0, 1, 4, 2, 3).reshape(B, 8 * nplanes, Hs, Ws)


def _phys_planes(plane0, n, x3):
    lps = range(plane0, plane0 + n)
    return sorted([_x3_plane(p) for p in lps] + [_x3_plane(p) + 4 for p in lps]) if x3 else list(lps)


def _conv_case(case):
    if isinstance(case, int):
        return _old_case(case) if case < NOLD else _random_case(case)
    return _forced_case(case)


@pytest.mark.parametrize("case", list(range(NOLD + NRANDOM)) + sorted(FORCED))
def test_conv_fuzz(case):
    from bin_b200 import ops
    spec, B, H, W, sub, x3, mag = _conv_case(case)
    prec = "x3" if x3 else "f16"
    label = _inst(spec)[0]
    resident = _resident(spec, x3)
    k, cin, cout, cout_pad, epi = spec["k"], spec["cin"], spec["cout"], spec["cout_pad"], spec["epi"]
    where = (case, label, prec, "resident" if resident else "streamed", spec.get("tag", ""), B, H, W, sub, mag)
    if isinstance(case, str) and case.startswith("many_"):
        assert _ntiles(spec, B, H, W, sub) > torch.cuda.get_device_properties(0).multi_processor_count, where
    if isinstance(case, str) and case.startswith(("res_", "stream_")):
        assert resident == case.startswith("res_"), where
    seed = case if isinstance(case, int) else 5000 + sorted(FORCED).index(case)
    g = torch.Generator(device=DEV).manual_seed(9000 + seed)
    rn = lambda *shape: torch.randn(shape, generator=g, device=DEV, dtype=torch.float64)
    opnd = (lambda t: t.float().double()) if x3 else (lambda t: t.half().double())   # the operand the kernel sees

    # ---- tensors: NaN everywhere, data on the planes a call reads, the sentinel on the planes it writes
    vals = {n: torch.full((B, 8 * p, H * f, W * f), NAN, dtype=torch.float64, device=DEV) for n, (p, f) in spec["tensors"].items()}
    nstore = spec["store"] or cout_pad // 8
    reads = list(spec["segs"]) + ([(spec["res"][0], spec["res"][1], nstore)] if spec["res"] else [])
    for name, p0, np_ in reads:
        blk = vals[name][:, 8 * p0:8 * (p0 + np_)]
        fill = torch.isnan(blk)
        blk[fill] = opnd(rn(*blk.shape) * mag)[fill]
    X = torch.cat([vals[n][:, 8 * p0:8 * (p0 + np_)] for n, p0, np_ in spec["segs"]], 1)
    if X.shape[1] > cin:                                  # SFENet1: the packer's zero channels past 12 n
        X[:, cin:] = 0
        n0, p0, np_ = spec["segs"][0]
        vals[n0][:, 8 * p0 + cin:8 * (p0 + np_)] = 0
    if epi == 0:
        on, op0 = spec["out"]
        vals[on][:, 8 * op0:8 * (op0 + nstore)] = SENTINEL
    elif epi == 1:
        on, op0 = spec["out"]
        vals[on][:, 8 * op0:8 * (op0 + 8)] = SENTINEL
    dev_t = {n: _to_device(v, x3) for n, v in vals.items()}
    before = {n: t.clone() for n, t in dev_t.items()}

    # ---- weights, bias, the launch
    w32 = (rn(cout, X.shape[1], k, k) / math.sqrt(cin * k * k)).float()
    if X.shape[1] > cin:
        w32[:, cin:] = 0
    b32 = (rn(cout) * 0.1 * mag).float()
    wp = ops.pack_conv_weight(w32, cout_pad, X.shape[1], variant=spec["variant"], prec=int(x3))
    bp = ops.pad_bias(b32, cout_pad)
    segs = spec["segs"]
    kw = dict(in0_plane0=segs[0][1], in0_planes=segs[0][2], relu=spec["relu"], epilogue=epi, variant=spec["variant"],
              sub=sub, store_planes=spec["store"], x3=x3)
    if len(segs) > 1:
        kw.update(in1=dev_t[segs[1][0]], in1_plane0=segs[1][1], in1_planes=segs[1][2])
    if epi != 2:
        kw.update(out=dev_t[spec["out"][0]], out_plane0=spec["out"][1])
    if spec["res"]:
        kw.update(res=dev_t[spec["res"][0]], res_plane0=spec["res"][1])
    outs, frames, table = [], [], None
    if epi == 2:
        fin = spec["final"]
        nc, nf, Bc = fin["ncalls"], fin["nframes"], fin["Bc"]
        npool = nc * (nf - 1) + 1 if fin["shared"] else nc * nf
        pool = [torch.rand((Bc, 3, H, W), generator=g, device=DEV) for _ in range(npool)]
        frames = [[pool[c * (nf - 1) + f] if fin["shared"] else pool[c * nf + f] for f in range(nf)] for c in range(nc)]
        outs = [torch.full((Bc, 3, H, W), SENTINEL, device=DEV) for _ in range(nc)]
        outs0 = [o.clone() for o in outs]
        kw["frames"] = table = ops.make_frames(frames, outs)
    ops.conv_fwd(dev_t[segs[0][0]], wp, bp, k, cout_pad, **kw)
    torch.cuda.synchronize()

    # ---- fp64 reference and per-element bar
    w64 = opnd(w32)
    wpad = torch.zeros((cout_pad,) + w64.shape[1:], dtype=torch.float64, device=DEV)
    wpad[:cout] = w64
    bpad = torch.zeros(cout_pad, dtype=torch.float64, device=DEV)
    bpad[:cout] = b32.double()
    ref = F.conv2d(X, wpad, bpad, padding=k // 2)
    if spec["relu"]:
        ref = ref.relu()
    A = F.conv2d(X.abs(), wpad.abs(), bpad.abs(), padding=k // 2)
    W1 = wpad.abs().sum((1, 2, 3)).view(1, -1, 1, 1)
    X1 = F.conv2d(X.abs(), torch.ones((1,) + w64.shape[1:], dtype=torch.float64, device=DEV), padding=k // 2)
    b0, nb, y0, ny = sub if sub else (0, B, 0, H)
    bsl, ysl = slice(b0, b0 + nb), slice(y0, y0 + ny)
    if epi == 0:
        rabs = torch.zeros_like(ref[:, :8 * nstore])
        ref = ref[:, :8 * nstore]
        A, W1 = A[:, :8 * nstore], W1[:, :8 * nstore]
        if spec["res"]:
            rn_, rp0 = spec["res"]
            r = vals[rn_][:, 8 * rp0:8 * (rp0 + nstore)]
            ref, rabs = ref + r, r.abs()
        on, op0 = spec["out"]
        got = _from_device(dev_t[on], op0, nstore, x3)
        sl = (bsl, slice(None), ysl)
        written = [(on, _phys_planes(op0, nstore, x3), bsl, ysl)]
    elif epi == 1:
        ref, A, rabs = F.pixel_shuffle(ref, 2), F.pixel_shuffle(A, 2), 0.0
        W1 = W1.max()                                      # bounds every sub-pixel channel
        X1 = X1.repeat_interleave(2, 2).repeat_interleave(2, 3)
        on, op0 = spec["out"]
        got = _from_device(dev_t[on], op0, 8, x3)
        sl = (bsl, slice(None), slice(2 * y0, 2 * (y0 + ny)))
        written = [(on, _phys_planes(op0, 8, x3), bsl, sl[2])]
    else:
        fin = spec["final"]
        nf, Bc = fin["nframes"], fin["Bc"]
        ref, A, W1, rabs = ref[:, :3], A[:, :3], W1[:, :3], 0.0
        fsum = torch.cat([sum(f.double() for f in fr) for fr in frames], 0)
        fabs = torch.cat([sum(f.double().abs() for f in fr) for fr in frames], 0)
        ref = ref + fsum / nf
        got = torch.cat([o.double() for o in outs], 0)
        sl = (bsl, slice(None), ysl)
        written = []
    if epi == 2:
        extra = ulp32(ref) + (nf + 1) * U * fabs
        bar = (C_X3 * U * A + 2.0 ** -22 * 3 * A + 2.0 ** -25 * W1 + 2.0 ** -33 * X1) + extra if x3 else C_FINAL * U * A + extra
    elif x3:
        bar = C_X3 * U * (A + rabs) + 2.0 ** -22 * (3 * A + ref.abs() + 2 * rabs) + 2.0 ** -25 * (W1 + 2) + 2.0 ** -33 * X1
    else:
        bar = ulp16(ref) + C_F16 * U * A
    err = (got - ref)[sl].abs()
    assert torch.isfinite(got[sl]).all(), ("non-finite output", where)
    ratio = (err / bar[sl]).max().item()
    _record(label, prec, ratio)
    print(f"[fwd fuzz] {case} {label} {prec} {'resident' if resident else 'streamed'} {spec.get('tag', '')} "
          f"B={B} H={H} W={W} sub={sub} mag={mag:g}: worst err/bar {ratio:.3f}")
    assert ratio <= 1.0, (where, ratio, err.max().item())

    # ---- nothing outside the written range changed: NaN planes, sentinels, inputs keep their bits
    for name, t in dev_t.items():
        keep = torch.ones(t.shape, dtype=torch.bool, device=DEV)
        for wn, planes, bs, ys in written:
            if wn == name:
                pl = torch.tensor(planes, device=DEV)
                m = torch.zeros(t.shape, dtype=torch.bool, device=DEV)
                m[bs, :, ys] = True
                pm = torch.zeros(t.shape[1], dtype=torch.bool, device=DEV)
                pm[pl] = True
                keep &= ~(m & pm.view(1, -1, 1, 1, 1))
        assert torch.equal(_bits(t)[keep], _bits(before[name])[keep]), ("wrote outside its range", name, where)
    if epi == 2:
        for c, (o, o0) in enumerate(zip(outs, outs0)):
            m = torch.ones(o.shape, dtype=torch.bool, device=DEV)
            for bb in range(Bc):
                if b0 <= c * Bc + bb < b0 + nb:
                    m[bb, :, ysl] = False
            assert torch.equal(_bits(o)[m], _bits(o0)[m]), ("final wrote outside its range", c, where)
    del table


# --------------------------------------------------------------------------------------------------------------------
# part 2: the fused RDB tail against fp64
# --------------------------------------------------------------------------------------------------------------------
TAIL = [  # (i, g0 = 16 i (training layout) or 0, B, H, W, sub)
    (1, False, 1, 4, 30, None), (5, True, 2, 5, 31, None), (11, True, 3, 9, 29, (1, 2, 3, 5)), (0, False, 2, 8, 61, None),
    (7, False, 1, 1, 1, None), (3, True, 3, 3, 59, (0, 1, 1, 2)), (9, False, 2, 13, 90, (1, 1, 0, 0)),
    (2, True, 1, 7, 2, None), (6, False, 3, 48, 130, None), (10, True, 3, 48, 130, (0, 3, 5, 40)),
]


@pytest.mark.parametrize("idx", range(len(TAIL)))
def test_rdb_tail_vs_fp64(idx):
    from bin_b200 import ops
    i, train, B, H, W, sub = TAIL[idx]
    g0 = 16 * i if train else 0
    where = (i, g0, B, H, W, sub)
    gen = torch.Generator(device=DEV).manual_seed(300 + idx)
    rn = lambda *shape: torch.randn(shape, generator=gen, device=DEV, dtype=torch.float64)
    b0, nb, y0, ny = (sub[0], sub[1] or B - sub[0], sub[2], sub[3] or H - sub[2]) if sub else (0, B, 0, H)
    if idx >= 8:
        tiles = nb * -(-ny // 4) * -(-W // 30)
        assert tiles > torch.cuda.get_device_properties(0).multi_processor_count, where
    cat = torch.full((B, 1152, H, W), NAN, dtype=torch.float64, device=DEV)
    gt = torch.full((B, 8 * 192, H, W), NAN, dtype=torch.float64, device=DEV)
    xp0, op0 = (12 * (i - 1), 12 * i) if i else (None, 0)
    if i:
        cat[:, 8 * xp0:8 * xp0 + 96] = rn(B, 96, H, W).half().double()
        x = cat[:, 8 * xp0:8 * xp0 + 96]
    else:
        xt = rn(B, 96, H, W).half().double()
        x = xt
    gt[:, 8 * g0:8 * g0 + 96] = rn(B, 96, H, W).half().double()
    cat[:, 8 * op0:8 * op0 + 96] = SENTINEL
    g012 = gt[:, 8 * g0:8 * g0 + 96]
    w3 = (rn(32, 192, 3, 3) / math.sqrt(1728)).float()
    wl = (rn(96, 224, 1, 1) / math.sqrt(224)).float()
    b3, bl = (rn(32) * 0.1).float(), (rn(96) * 0.1).float()
    dcat, dg = _to_device(cat, False), _to_device(gt, False)
    dx = dcat if i else _to_device(xt, False)
    before = [dcat.clone(), dg.clone(), dx.clone()]
    ops.rdb_tail_fwd(dx, dg, ops.pack_conv_weight(w3, 32, 192), b3.to(DEV), ops.pack_conv_weight(wl, 96, 224), bl.to(DEV),
                     dcat, x_plane0=xp0 or 0, g_plane0=g0, out_plane0=op0, sub=sub or (0, 0, 0, 0))
    torch.cuda.synchronize()
    w3d, wld = w3.half().double(), wl.half().double()
    in3 = torch.cat((x, g012), 1)
    pre3 = F.conv2d(in3, w3d, b3.double(), padding=1)
    A3 = F.conv2d(in3.abs(), w3d.abs(), b3.double().abs(), padding=1)
    g3 = pre3.relu().half().double()                       # the kernel's g3 tile is fp16
    inl = torch.cat((x, g012, g3), 1)
    ref = F.conv2d(inl, wld, bl.double()) + x
    A = F.conv2d(inl.abs(), wld.abs(), bl.double().abs()) + x.abs()
    g3_err = ulp16(g3) + C_TAIL * U * A3
    bar = ulp16(ref) + C_F16 * U * A + F.conv2d(g3_err, wld[:, 192:].abs())
    got = _from_device(dcat, op0, 12, False)
    sl = (slice(b0, b0 + nb), slice(None), slice(y0, y0 + ny))
    assert torch.isfinite(got[sl]).all(), where
    ratio = ((got - ref)[sl].abs() / bar[sl]).max().item()
    _record("rdb_tail", "f16", ratio)
    print(f"[fwd fuzz] rdb_tail i={i} g0={g0} B={B} H={H} W={W} sub={sub}: worst err/bar {ratio:.3f}")
    assert ratio <= 1.0, (where, ratio)
    keep = torch.ones(dcat.shape, dtype=torch.bool, device=DEV)
    keep[sl[0], op0:op0 + 12, sl[2]] = False
    assert torch.equal(_bits(dcat)[keep], _bits(before[0])[keep]), ("tail wrote outside its range", where)
    assert torch.equal(_bits(dg), _bits(before[1])), where
    if not i:
        assert torch.equal(_bits(dx), _bits(before[2])), where


# --------------------------------------------------------------------------------------------------------------------
# part 3: the frame packer, bit for bit
# --------------------------------------------------------------------------------------------------------------------
PACK = [  # (ncalls, Bc, nframes, shared, H, W)
    (1, 1, 2, False, 2, 2), (2, 3, 3, True, 70, 62), (6, 1, 2, True, 64, 128), (3, 2, 5, True, 66, 130),
    (4, 1, 3, False, 10, 98), (5, 1, 5, True, 2, 258), (1, 3, 5, False, 130, 4), (6, 2, 3, True, 46, 46),
]


@pytest.mark.parametrize("x3", [False, True])
@pytest.mark.parametrize("idx", range(len(PACK)))
def test_pack_frames_bit_exact(idx, x3):
    import ctypes as C
    from bin_b200 import ops
    from bin_b200._lib import check, lib
    nc, Bc, nf, shared, H, W = PACK[idx]
    gen = torch.Generator(device=DEV).manual_seed(400 + idx)
    npool = nc * (nf - 1) + 1 if shared else nc * nf
    pool = [torch.randn((Bc, 3, H, W), generator=gen, device=DEV) * 3 for _ in range(npool)]
    frames = [[pool[c * (nf - 1) + f] if shared else pool[c * nf + f] for f in range(nf)] for c in range(nc)]
    cin_pad = (12 * nf + 31) // 32 * 32
    dst = torch.full((nc * Bc, cin_pad // 8 * (2 if x3 else 1), H // 2, W // 2, 8), NAN, dtype=torch.float16, device=DEV)
    fr = ops.make_frames(frames, [None] * nc)
    check(lib().bin_pack_frames_p(C.byref(fr), H, W, ops.act_view(dst), int(x3), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    # pixel_reshuffle(cat(frames), 2) (RDN.py:107-132): channel (f*3+rgb)*4 + dy*2 + dx, zero-padded to cin_pad
    v = torch.zeros((nc * Bc, cin_pad, H // 2, W // 2), device=DEV)
    for c in range(nc):
        x = torch.cat(frames[c], 1)
        v[c * Bc:(c + 1) * Bc, :12 * nf] = x.reshape(Bc, 3 * nf, H // 2, 2, W // 2, 2).permute(0, 1, 3, 5, 2, 4).reshape(
            Bc, 12 * nf, H // 2, W // 2)
    p8 = v.view(nc * Bc, cin_pad // 8, 8, H // 2, W // 2).permute(0, 1, 3, 4, 2)
    hi = p8.half()
    if not x3:
        assert torch.equal(_bits(dst), _bits(hi.contiguous()))
        assert torch.equal(_bits(ops.pack_frames(frames)), _bits(hi.contiguous()))
        return
    lo = (p8 - hi.float()).half()
    for lp in range(cin_pad // 8):
        assert torch.equal(_bits(dst[:, _x3_plane(lp)]), _bits(hi[:, lp].contiguous())), ("hi", lp)
        assert torch.equal(_bits(dst[:, _x3_plane(lp) + 4]), _bits(lo[:, lp].contiguous())), ("lo", lp)
    assert torch.equal(_bits(ops.pack_frames(frames, prec=1)), _bits(dst))


# --------------------------------------------------------------------------------------------------------------------
# part 4: the ConvLSTM cell against fp64
# --------------------------------------------------------------------------------------------------------------------
def _convlstm_launch(cells, B, H, W, write_c):
    """One bin_convlstm_fwd launch over the cell table [(x, w, b, c_prev, h_prev), ...] -> ([h], [c]), both NaN-filled
    beforehand; write_c False passes c_out NULL."""
    from bin_b200 import _lib
    P = lambda t: None if t is None else t.data_ptr()
    hs = [torch.full((B, 3, H, W), NAN, device=DEV) for _ in cells]
    cs = [torch.full((B, 3, H, W), NAN, device=DEV) for _ in cells]
    tab = (_lib.LstmCell * len(cells))(*[_lib.LstmCell(x.data_ptr(), P(cp), P(hp), w.data_ptr(), b.data_ptr(), h.data_ptr(),
                                                       c.data_ptr() if write_c else None)
                                         for (x, w, b, cp, hp), h, c in zip(cells, hs, cs)])
    _lib.check(_lib.lib().bin_convlstm_fwd(tab, len(cells), B, H, W, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return hs, cs


@pytest.mark.parametrize("ncells", [1, 2, 3])
@pytest.mark.parametrize("W", [1, 2, 3, 4, 5, 63, 64, 65, 67, 128, 130])
def test_convlstm_vs_fp64(W, ncells):
    """ncells cells in one launch, each with its own inputs and weights: every cell against fp64, and with more than one
    cell every cell with the bits of its own one-cell launch."""
    gen = torch.Generator(device=DEV).manual_seed(500 + W)
    worst = 0.0
    for hi_, H in enumerate([1, 2, 15, 16, 17, 33]):
        for mode in ("none", "state", "state_no_c"):
            B = 1 + (hi_ + len(mode)) % 3
            state = mode != "none"
            cells = []
            for _ in range(ncells):
                x = torch.randn((B, 3, H, W), generator=gen, device=DEV) * 3
                w = torch.randn((12, 6, 3, 3), generator=gen, device=DEV) * 2      # gate sums reach +-30 and beyond
                b = torch.randn((12,), generator=gen, device=DEV)
                cp = (torch.rand((B, 3, H, W), generator=gen, device=DEV) * 100 - 50) if state else None
                hp = (torch.rand((B, 3, H, W), generator=gen, device=DEV) * 2 - 1) if state else None
                cells.append((x, w, b, cp, hp))
            hs, cs = _convlstm_launch(cells, B, H, W, mode != "state_no_c")
            for k, ((x, w, b, cp, hp), h, c) in enumerate(zip(cells, hs, cs)):
                c0 = cp.double() if state else torch.zeros((B, 3, H, W), dtype=torch.float64, device=DEV)
                h0 = hp.double() if state else torch.zeros_like(c0)
                xh = torch.cat((x.double(), h0), 1)
                gsum = F.conv2d(xh, w.double(), b.double(), padding=1)
                G = F.conv2d(xh.abs(), w.double().abs(), b.double().abs(), padding=1)
                gi, gj, gf, go = gsum.chunk(4, 1)
                Gi, Gj, Gf, Go = G.chunk(4, 1)
                si, tj, sf, so = torch.sigmoid(gi), torch.tanh(gj), torch.sigmoid(gf + 1.0), torch.sigmoid(go)
                c_ref = c0 * sf + si * tj
                h_ref = torch.tanh(c_ref) * so
                e_i, e_f, e_o = (0.25 * K_LSTM * U * G_ + T_LSTM for G_ in (Gi, Gf + 1.0, Go))
                e_j = K_LSTM * U * Gj + T_LSTM
                e_c = c0.abs() * e_f + tj.abs() * e_i + si.abs() * e_j + 3 * U * (c0 * sf).abs() + 3 * U * (si * tj).abs()
                e_h = so.abs() * (e_c + T_LSTM) + torch.tanh(c_ref).abs() * e_o + U * h_ref.abs()
                rh = ((h.double() - h_ref).abs() / e_h).max().item()
                worst = max(worst, rh)
                assert rh <= 1.0, (mode, B, H, W, k, rh)
                if mode == "state_no_c":
                    assert torch.isnan(c).all()                           # c_out NULL: nothing written
                else:
                    rc = ((c.double() - c_ref).abs() / e_c).max().item()
                    worst = max(worst, rc)
                    assert rc <= 1.0, (mode, B, H, W, k, rc)
                if ncells > 1:
                    (h1,), (c1,) = _convlstm_launch([cells[k]], B, H, W, mode != "state_no_c")
                    assert torch.equal(_bits(h), _bits(h1)) and torch.equal(_bits(c), _bits(c1)), (mode, B, H, W, k)
    _record("convlstm", "f32", worst)
    print(f"[fwd fuzz] convlstm W={W} cells={ncells}: worst err/bar {worst:.3f}")
