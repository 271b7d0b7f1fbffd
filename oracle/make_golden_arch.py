"""Generate the fixtures of the G0 / D backbone configurations by EXECUTING THE UNMODIFIED REFERENCE (laomao0/BIN).

Run in the authoring container only (needs /root/reference):

    python oracle/make_golden_arch.py

The reference builds every backbone class from a width G0 and a depth D (RDN.py:167-334): G0 = 64, D = 6 by default,
G0 = 96, D = 12 in bin_stage4_lstm (RDN.py:418).  This script pins ``oracle/arch_oracle.py`` at the other
configurations the library runs, as ``make_golden.py`` pins ``oracle/bin_oracle.py`` at the shipped one:

  tests/golden/arch_backbones.npz   the three backbone classes at (G0, D) = (64, 6), (64, 12), (96, 6)
  tests/golden/arch_window.npz      a six-frame window whose .model is RDN_residual_interp_5_input(lstm=True, GO=64,
                                    D=6), at 64x96: its 14 outputs
  tests/golden/arch_window_grad.npz the same window at 16x16: d(sum_k <out_k, cot_k>) / d(frames, a few parameters)
  tests/golden/arch_schema.json     the reference's state_dict keys and shapes for each of these configurations

Weights are ``arch_oracle.synth_backbone_sd`` / ``synth_state_dict(seed, G0, D)`` loaded with ``strict=True``; inputs are
``bin_oracle.synth_frames``.  Nothing under /root/reference is copied; only tensors it computes are stored.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, "/root/reference")

import models.archs.RDN as R          # noqa: E402  (the reference itself)
from oracle import arch_oracle as A  # noqa: E402
from oracle import bin_oracle as O    # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
torch.set_num_threads(os.cpu_count())

CONFIGS = [(64, 6), (64, 12), (96, 6)]
CLASSES = {2: "RDN_residual_interp_2_input", 3: "RDN_residual_interp_2_1_input", 5: "RDN_residual_interp_4_1_input"}
BACKBONE_SHAPE = (2, 20, 36)          # B, H, W: odd tile remainders in both directions
WINDOW_ARCH = (64, 6)
WINDOW_SHAPE = (1, 64, 96)
GRAD_SHAPE = (1, 16, 16)
GRAD_PARAMS = ["model.model1_1.SFENet1.weight", "model.model1_1.RDBs.0.convs.0.conv.0.weight",
               "model.model2_1.RDBs.5.LFF.weight", "model.model3_1.GFF.0.weight", "model.model4_1.UPNet.0.bias",
               "clstm_4_prime.Gates.weight"]


def backbone_seed(n, g0, d):
    return 500 + 100 * n + g0 + d


def save(name, **arrs):
    np.savez_compressed(os.path.join(OUT, name), **{k: np.asarray(v) for k, v in arrs.items()})
    print("wrote", name, len(arrs), "arrays")


def schema(module):
    return [[k, list(v.shape)] for k, v in module.state_dict().items()]


def light_window():
    g0, d = WINDOW_ARCH
    net = R.bin_stage4_lstm()
    net.model = R.RDN_residual_interp_5_input(lstm=True, GO=g0, D=d)       # the line that builds it in the reference
    sd = A.synth_state_dict(0, g0, d)
    res = net.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert list(net.state_dict().keys()) == list(sd.keys()), "key ORDER differs from reference"
    return net.eval()


def main():
    shapes = {}
    outs = {}
    B, H, W = BACKBONE_SHAPE
    for g0, d in CONFIGS:
        for n, cls in CLASSES.items():
            m = getattr(R, cls)(G0=g0, D=d).eval()
            sd = A.synth_backbone_sd(n, backbone_seed(n, g0, d), g0, d)
            res = m.load_state_dict(sd, strict=True)
            assert not res.missing_keys and not res.unexpected_keys
            assert list(m.state_dict().keys()) == list(sd.keys())
            shapes[f"{cls}/{g0}/{d}"] = schema(m)
            fr = O.synth_frames(n, B, H, W, seed=backbone_seed(n, g0, d) + 1)
            with torch.no_grad():
                outs[f"{n}_{g0}_{d}"] = m(*fr).numpy()
    save("arch_backbones.npz", meta=np.array(BACKBONE_SHAPE), **outs)

    net = light_window()
    shapes[f"window/{WINDOW_ARCH[0]}/{WINDOW_ARCH[1]}"] = schema(net)
    B, H, W = WINDOW_SHAPE
    fr = O.synth_frames(6, B, H, W, seed=4321)
    with torch.no_grad():
        wo = net(*fr)
    save("arch_window.npz", meta=np.array([B, H, W, 4321, 0]), **{f"out{k}": o.numpy() for k, o in enumerate(wo)})

    net.train()
    B, H, W = GRAD_SHAPE
    fr = [f.requires_grad_(True) for f in O.synth_frames(6, B, H, W, seed=19)]
    wo = net(*fr)
    cots = O.synth_frames(14, B, H, W, seed=20)
    loss = sum((o * (c - 0.5)).sum() for o, c in zip(wo, cots))
    params = dict(net.named_parameters())
    grads = torch.autograd.grad(loss, fr + [params[k] for k in GRAD_PARAMS])
    save("arch_window_grad.npz", meta=np.array([B, H, W, 19, 20]), loss=loss.detach().numpy(),
         **{f"dframe{k}": g.numpy() for k, g in enumerate(grads[:6])},
         **{"d:" + k: g.numpy() for k, g in zip(GRAD_PARAMS, grads[6:])})

    with open(os.path.join(OUT, "arch_schema.json"), "w") as fh:
        json.dump(shapes, fh, separators=(",", ":"))
        fh.write("\n")
    print("wrote arch_schema.json", len(shapes), "modules")


if __name__ == "__main__":
    main()
