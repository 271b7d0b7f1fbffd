"""TEST INFRASTRUCTURE: the backward convs of one backbone as run_backbone_bwd (bin_b200/csrc/api.cu) launches them.

A backbone of width G0 and depth D keeps its G0-channel feature maps in P = G0 / 8 planes of 8 channels: f1, f2, t1,
t2 and their gradients take P planes, cat and dcat (the D RDB outputs) P D planes, the growth maps 16 D planes (16 in
recompute mode, where only the current RDB's are rebuilt), their gradient dg 16 planes, and the packed frames x0 and
their gradient 4 or 8 planes.  Each conv's data gradient runs as one or two launches of the forward conv kernel over dY
with transposed weights (bin_pack_conv_weight_t): rows [row0, row0 + nrows) of the forward conv's Cin axis, padded to a
multiple of 96 and clipped to `store` output planes.

spec(kind, rnd, g0, d, **force) describes one of them; backbone_layers(nframes, g0, d) lists the (kind, force) of every
conv of a backbone in the library's conv order (nn.Module registration order, RDN.py:187-208).
"""
from __future__ import annotations

from typing import Dict, List, Tuple


def spec(kind: str, rnd, g0: int = 96, d: int = 12, **force) -> Dict:
    """One backward conv.  x: input segments (tensor planes, plane0, planes); dy: (tensor planes, plane0) of the dY
    range; dgrad: data-gradient launches, out = (tensor planes, plane0, store_planes) with tensor planes None when the
    output lives in the dY tensor itself.  Choices not forced are drawn from rnd, in an order that gives G0 = 96, D = 12
    the draws it always had.  force recompute=True puts the growth maps of an RDB conv or LFF at plane 0 of a 16-plane
    tensor, as the recomputing backward rebuilds them."""
    pick = lambda key, choices: force[key] if key in force else rnd.choice(choices)
    P = g0 // 8
    growth = lambda i: (16, 0) if force.get("recompute") else (16 * d, 16 * i)
    if kind == "sfe1":                      # SFENet1 5x5 (12 n) -> G0; x0 = the packed frames, 4 or 8 planes
        cin = pick("cin", [24, 36, 60])
        xp = (cin + 31) // 32 * 4
        return dict(cin=cin, cout=g0, k=5, x=[(xp, 0, xp)], dy=(P, 0), dgrad=[dict(row0=0, nrows=cin, out=(xp, 0, xp), acc=False)],
                    tag=f"g0={g0}")
    if kind in ("sfe2", "gff1"):            # SFENet2 (dgrad accumulates into d f1) / GFF.1 (dgrad overwrites d t1)
        acc = pick("acc", [False, True]) if kind == "sfe2" else False
        return dict(cin=g0, cout=g0, k=3, x=[(P, 0, P)], dy=(P, 0), dgrad=[dict(row0=0, nrows=g0, out=(P, 0, P), acc=acc)],
                    tag=f"g0={g0}")
    if kind == "rdb":                       # conv c of RDB i: x-stacked wgrad, dY = planes [4c, 4c+4) of the growth grads
        c, i = pick("c", range(4)), pick("i", range(d))
        xin = (P * d, P * (i - 1), P) if i else (P, 0, P)
        dg = [dict(row0=0, nrows=g0, out=xin, acc=True)]
        if c:                               # growth rows accumulate in place into planes [0, 4c) of the dY tensor
            dg.append(dict(row0=g0, nrows=32 * c, out=(None, 0, 4 * c), acc=True))
        return dict(cin=g0 + 32 * c, cout=32, k=3, x=[xin] + ([(*growth(i), 4 * c)] if c else []), dy=(16, 4 * c), dgrad=dg,
                    tag=f"g0={g0} d={d} c={c} i={i}")
    if kind == "lff":                       # LFF 1x1 (G0 + 128) -> G0 of RDB i: dY = d x_{i+1} at planes P i of d cat
        i = pick("i", range(d))
        xin = (P * d, P * (i - 1), P) if i else (P, 0, P)
        dx = (None, P * (i - 1), P) if i else (P, 0, P)
        return dict(cin=g0 + 128, cout=g0, k=1, x=[xin, (*growth(i), 16)], dy=(P * d, P * i),
                    dgrad=[dict(row0=0, nrows=g0, out=dx, acc=True), dict(row0=g0, nrows=128, out=(16, 0, 16), acc=False)],
                    tag=f"g0={g0} d={d} i={i}")
    if kind == "gff0":                      # GFF.0 1x1 D G0 -> G0: channel tiles of 128 in the wgrad
        return dict(cin=g0 * d, cout=g0, k=1, x=[(P * d, 0, P * d)], dy=(P, 0),
                    dgrad=[dict(row0=0, nrows=g0 * d, out=(P * d, 0, P * d), acc=False)], tag=f"g0={g0} d={d}")
    if kind == "up0":                       # UPNet.0 3x3 G0 -> 256: N = 256, one tap per wgrad launch
        return dict(cin=g0, cout=256, k=3, x=[(P, 0, P)], dy=(32, 0), dgrad=[dict(row0=0, nrows=g0, out=(P, 0, P), acc=False)],
                    tag=f"g0={g0}")
    if kind == "up2":                       # UPNet.2 3x3 64 -> 3: N = 16, dY channels 3..31 zero
        return dict(cin=64, cout=3, k=3, x=[(8, 0, 8)], dy=(4, 0), dgrad=[dict(row0=0, nrows=64, out=(8, 0, 8), acc=False)])
    if kind == "ring":                      # 5x5 with 128 < Cout <= 256: a one-stage wgrad ring (no backbone conv)
        return dict(cin=36, cout=200, k=5, x=[(8, 0, 8)], dy=(28, 0), dgrad=[dict(row0=0, nrows=36, out=(8, 0, 8), acc=False)])
    raise ValueError(kind)


def backbone_layers(nframes: int, g0: int, d: int) -> List[Tuple[str, Dict]]:
    """(kind, forced choices) of every conv of a backbone, in the library's conv order: SFENet1, SFENet2, the four growth
    convs and the LFF of each RDB, GFF.0, GFF.1, UPNet.0, UPNet.2."""
    out = [("sfe1", dict(cin=12 * nframes)), ("sfe2", dict(acc=True))]
    for i in range(d):
        out += [("rdb", dict(c=c, i=i)) for c in range(4)] + [("lff", dict(i=i))]
    return out + [("gff0", {}), ("gff1", {}), ("up0", {}), ("up2", {})]
