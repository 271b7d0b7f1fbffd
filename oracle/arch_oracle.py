"""CPU oracle of the backbones at any width G0 and depth D -- TEST INFRASTRUCTURE ONLY.

The reference builds every backbone class from a width G0 and a depth D (``models/archs/RDN.py:167-334``): G0 = 64,
D = 6 by default, G0 = 96, D = 12 in ``bin_stage4_lstm`` (RDN.py:418).  ``bin_oracle`` restates the shipped
configuration; this module restates the schema, the synthetic weights, the backbone and the window for any (G0, D),
with the per-layer arithmetic of ``bin_oracle`` (``conv``, ``rdb``, ``convlstm``, ``space_to_depth2`` and its fp16
storage emulation).  At G0 = 96, D = 12 every function here gives what its ``bin_oracle`` namesake gives.  It is pinned
to the reference by ``oracle/make_golden_arch.py`` and ``tests/test_arch_cpu.py``.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import torch

from . import bin_oracle as O

Tensor = torch.Tensor
SD = O.SD


def backbone_param_shapes(nframes: int, G0: int = O.G0, D: int = O.D) -> List[Tuple[str, Tuple[int, ...]]]:
    """(suffix, shape) for one backbone of width G0 and depth D, in the reference's registration order
    (RDN.py:187-208 / 245-266 / 299-320)."""
    C, G = O.C, O.G
    out: List[Tuple[str, Tuple[int, ...]]] = []
    out += [("SFENet1.weight", (G0, 12 * nframes, 5, 5)), ("SFENet1.bias", (G0,))]
    out += [("SFENet2.weight", (G0, G0, 3, 3)), ("SFENet2.bias", (G0,))]
    for i in range(D):
        for c in range(C):
            out += [(f"RDBs.{i}.convs.{c}.conv.0.weight", (G, G0 + c * G, 3, 3)),
                    (f"RDBs.{i}.convs.{c}.conv.0.bias", (G,))]
        out += [(f"RDBs.{i}.LFF.weight", (G0, G0 + C * G, 1, 1)), (f"RDBs.{i}.LFF.bias", (G0,))]
    out += [("GFF.0.weight", (G0, D * G0, 1, 1)), ("GFF.0.bias", (G0,))]
    out += [("GFF.1.weight", (G0, G0, 3, 3)), ("GFF.1.bias", (G0,))]
    out += [("UPNet.0.weight", (256, G0, 3, 3)), ("UPNet.0.bias", (256,))]
    out += [("UPNet.2.weight", (3, 64, 3, 3)), ("UPNet.2.bias", (3,))]
    return out


def synth_backbone_sd(nframes: int, seed: int, G0: int = O.G0, D: int = O.D) -> SD:
    """bin_oracle.synth_backbone_sd at width G0 and depth D: U(+-1/sqrt(fan_in)) drawn in registration order."""
    gen = torch.Generator().manual_seed(seed)
    sd: SD = {}
    fan_in = 1
    for name, shape in backbone_param_shapes(nframes, G0, D):
        if name.endswith("weight"):
            fan_in = shape[1] * shape[2] * shape[3]
        sd[name] = O._uniform(shape, 1.0 / math.sqrt(fan_in), gen)
    return sd


def synth_state_dict(seed: int = 0, G0: int = O.G0, D: int = O.D) -> SD:
    """bin_oracle.synth_state_dict for the window whose ``.model`` is ``RDN_residual_interp_5_input(lstm=True, GO=G0,
    D=D)``: the same draws in the same order, aliases sharing storage."""
    sd: SD = {}
    gen = torch.Generator().manual_seed(seed * 1000 + 7)
    for n in O.LSTM_NAMES:
        bound = math.sqrt(6.0 / (6 * 9 + 12 * 9))
        sd[f"{n}.Gates.weight"] = O._uniform((12, 6, 3, 3), bound, gen)
        sd[f"{n}.Gates.bias"] = O._uniform((12,), 0.1, gen)
    for k, (canon, aliases) in enumerate(O.BACKBONE_ALIASES.items()):
        bsd = synth_backbone_sd(O.BACKBONE_NFRAMES[canon], seed * 1000 + 100 + k, G0, D)
        for a in aliases:
            for name, t in bsd.items():
                sd[f"model.{a}.{name}"] = t
    return sd


def backbone_depth(sd: SD) -> int:
    """D of a backbone state_dict: its number of residual dense blocks (every conv reads G0 off its weight's shape)."""
    return sum(1 for k in sd if k.startswith("RDBs.") and k.endswith(".LFF.weight"))


def backbone(frames: Sequence[Tensor], sd: SD) -> Tensor:
    """bin_oracle.backbone (RDN.py:210-222 / 268-280 / 322-334) at the G0 and D of `sd`."""
    q = O._q
    x0 = q(O.space_to_depth2(torch.cat(list(frames), 1)))                  # :211
    f1 = q(O.conv(x0, sd, "SFENet1"))                                      # :212
    x = q(O.conv(f1, sd, "SFENet2"))                                       # :213
    outs = []
    for i in range(backbone_depth(sd)):                                    # :215-217
        x = O.rdb(x, sd, f"RDBs.{i}")
        outs.append(x)
    x = q(O.conv(q(O.conv(torch.cat(outs, 1), sd, "GFF.0")), sd, "GFF.1") + f1)   # :218-219
    up = q(torch.nn.functional.pixel_shuffle(O.conv(x, sd, "UPNet.0"), 2))      # :205-206
    y = O.conv(up, sd, "UPNet.2")                                          # :207
    return y + sum(frames) / float(len(frames))                            # :221 / :279 / :333


def pyramid(fr: Sequence[Tensor], prev: Sequence[Optional[Tensor]], sd: SD) -> List[Tensor]:
    """bin_oracle.pyramid (RDN.py:367-405, lstm branch) with this module's backbone."""
    B1, B3, B5, B7, B9 = fr
    m1, m2, m3, m4 = (O.sub_sd(sd, k) for k in ("model1_1", "model2_1", "model3_1", "model4_1"))
    I2 = backbone((B1, B3), m1); I4 = backbone((B3, B5), m1)
    I6 = backbone((B5, B7), m1); I8 = backbone((B7, B9), m1)
    if prev[0] is not None:
        p4, p6, p8, p5, p7, p6b = prev
        I3 = backbone((p4, I2, I4), m2); I5 = backbone((p6, I4, I6), m2); I7 = backbone((p8, I6, I8), m2)
        I4b = backbone((p5, B3, I3, I5, B5), m3); I6b = backbone((p7, B5, I5, I7, B7), m3)
        I5c = backbone((p6b, I4, I4b, I6b, I6), m4)
    else:
        I3 = backbone((I2, I2, I4), m2); I5 = backbone((I4, I4, I6), m2); I7 = backbone((I6, I6, I8), m2)
        I4b = backbone((I3, B3, I3, I5, B5), m3); I6b = backbone((I5, B5, I5, I7, B7), m3)
        I5c = backbone((I4, I4, I4b, I6b, I6), m4)
    return [I2, I4, I6, I8, I3, I5, I7, I4b, I6b, I5c]


def window_forward(frames: Sequence[Tensor], sd: SD) -> List[Tensor]:
    """bin_oracle.window_forward (RDN.py:422-465) with this module's pyramid: 14 outputs."""
    assert len(frames) == 6
    msd = O.sub_sd(sd, "model")
    prev: List[Optional[Tensor]] = [None] * 6
    res = []
    for step in range(2):
        out = pyramid(frames[step:step + 5], prev, msd)
        hid = [out[1], out[2], out[3], out[5], out[6], out[8]]
        prev = [O.convlstm(hid[k], sd, O.LSTM_NAMES[k], None)[0] for k in range(6)] if step == 0 else prev
        res.append(out)
    r0, r1 = res
    return r0[:10] + [r1[3], r1[6], r1[8], r1[9]]
