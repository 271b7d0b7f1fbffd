"""CPU checks of the backbone configurations G0 in {64, 96}, 1 <= D <= 12 (the reference's RDN.py builds every backbone
class from a width G0 and a depth D): the state_dict schema against the reference's, the oracle against fixtures the
reference computed (oracle/make_golden_arch.py), the library's size queries against layouts computed here by hand, and
the refusal of every other configuration before anything is launched."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import arch_oracle as A
from oracle import bin_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 2e-6
CONFIGS = [(64, 6), (64, 12), (96, 6)]
CLASSES = {2: "RDN_residual_interp_2_input", 3: "RDN_residual_interp_2_1_input", 5: "RDN_residual_interp_4_1_input"}


def _seed(n, g0, d):                      # oracle/make_golden_arch.py
    return 500 + 100 * n + g0 + d


def _arch(n, g0, d):
    from bin_b200 import _lib
    return _lib.backbone_arch(n, g0, d)


def _schema(module):
    return [[k, list(v.shape)] for k, v in module.state_dict().items()]


@pytest.fixture(scope="module")
def ref_schema(golden_dir):
    with open(os.path.join(golden_dir, "arch_schema.json")) as fh:
        return json.load(fh)


# ------------------------------------------------------------------ the reference's schema, key for key
@pytest.mark.parametrize("g0,d", CONFIGS)
@pytest.mark.parametrize("n", sorted(CLASSES))
def test_backbone_state_dict_schema_matches_reference(ref_schema, n, g0, d):
    from bin_b200 import rdn
    m = getattr(rdn, CLASSES[n])(G0=g0, D=d)
    assert _schema(m) == ref_schema[f"{CLASSES[n]}/{g0}/{d}"]
    assert m.nconv == 5 * d + 6 and len(m._conv_params()) == 2 * m.nconv
    sd = A.synth_backbone_sd(n, 0, g0, d)
    assert list(sd) == [k for k, _ in _schema(m)]
    m.load_state_dict(sd, strict=True)


def test_light_window_state_dict_schema_matches_reference(ref_schema):
    """net.model = RDN_residual_interp_5_input(lstm=True, GO=64, D=6): the line that builds the light window in the
    reference gives the reference's keys and shapes here too, and the oracle's weights load strictly."""
    from bin_b200 import rdn
    net = rdn.bin_stage4_lstm()
    net.model = rdn.RDN_residual_interp_5_input(lstm=True, GO=64, D=6)
    assert _schema(net) == ref_schema["window/64/6"]
    net.load_state_dict(A.synth_state_dict(0, 64, 6), strict=True)


def test_default_arguments_are_the_references():
    """RDN.py's defaults are G0 = 64, D = 6 for every backbone class and the pyramid; bin_stage4_lstm stays 96 / 12."""
    from bin_b200 import rdn
    for cls in CLASSES.values():
        m = getattr(rdn, cls)()
        assert (m.G0, m.D) == (64, 6)
    pyr = rdn.RDN_residual_interp_5_input(lstm=True)
    assert (pyr.model1_1.G0, pyr.model1_1.D) == (64, 6)
    net = rdn.bin_stage4_lstm()
    assert (net.model.model4_1.G0, net.model.model4_1.D) == (96, 12) and net.model.model4_1.arch == 5


# ------------------------------------------------------------------ the oracle against the reference
def test_oracle_backbones_match_reference_fixtures(golden_dir):
    g = np.load(os.path.join(golden_dir, "arch_backbones.npz"))
    B, H, W = [int(v) for v in g["meta"]]
    for g0, d in CONFIGS:
        for n in CLASSES:
            sd = A.synth_backbone_sd(n, _seed(n, g0, d), g0, d)
            fr = O.synth_frames(n, B, H, W, seed=_seed(n, g0, d) + 1)
            out = A.backbone(fr, sd)
            assert (out - torch.from_numpy(g[f"{n}_{g0}_{d}"])).abs().max().item() <= TOL, (n, g0, d)


def test_oracle_light_window_matches_reference_fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "arch_window.npz"))
    B, H, W, seed, _ = [int(v) for v in g["meta"]]
    outs = A.window_forward(O.synth_frames(6, B, H, W, seed=seed), A.synth_state_dict(0, 64, 6))
    for k, o in enumerate(outs):
        assert (o - torch.from_numpy(g[f"out{k}"])).abs().max().item() <= TOL, k


def test_oracle_light_window_gradients_match_reference_fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "arch_window_grad.npz"))
    B, H, W, s_in, s_cot = [int(v) for v in g["meta"]]
    sd = {k: v.clone().requires_grad_(True) for k, v in A.synth_state_dict(0, 64, 6).items()}
    fr = [f.requires_grad_(True) for f in O.synth_frames(6, B, H, W, seed=s_in)]
    outs = A.window_forward(fr, sd)
    cots = O.synth_frames(14, B, H, W, seed=s_cot)
    loss = sum((o * (c - 0.5)).sum() for o, c in zip(outs, cots))
    names = [k[2:] for k in g.files if k.startswith("d:")]
    # the reference's aliases (model1_2 = model1_1, ...) share one tensor; the oracle's state dict holds the same object
    grads = torch.autograd.grad(loss, fr + [sd[n] for n in names])
    assert abs(loss.item() - float(g["loss"])) <= 1e-4 * max(1.0, abs(float(g["loss"])))
    for k in range(6):
        ref = torch.from_numpy(g[f"dframe{k}"])
        assert (grads[k] - ref).abs().max().item() <= 1e-5 * max(1.0, ref.abs().max().item()), k
    for n, gr in zip(names, grads[6:]):
        ref = torch.from_numpy(g["d:" + n])
        assert (gr - ref).abs().max().item() <= 1e-5 * max(1.0, ref.abs().max().item()), n


# ------------------------------------------------------------------ size queries against hand-computed layouts
def _align(v, a):
    return (v + a - 1) // a * a


def _convs(n, g0, d):
    """(cin, cout, ks, cout_pad) of each conv, registration order (RDN.py:187-208)."""
    out = [(12 * n, g0, 5, g0), (g0, g0, 3, g0)]
    for _ in range(d):
        out += [(g0 + 32 * c, 32, 3, 32) for c in range(4)] + [(g0 + 128, g0, 1, g0)]
    return out + [(d * g0, g0, 1, g0), (g0, g0, 3, g0), (g0, 256, 3, 256), (64, 3, 3, 16)]


def _packed_bytes(n, g0, d, x3=0):
    off = 0
    for cin, _, ks, cp in _convs(n, g0, d):
        off = _align(off + cp * _align(cin, 32) * ks * ks * 2 * (3 if x3 else 1), 256)
        off = _align(off + cp * 4, 256)
    return off


def _packed_t_bytes(n, g0, d):
    off = 0
    for i, (cin, cout, ks, _) in enumerate(_convs(n, g0, d)):
        parts = [g0, cin - g0] if 2 <= i < 2 + 5 * d else [cin]
        for rows in parts:
            if rows > 0:
                off = _align(off + _align(rows, 96) * _align(cout, 32) * ks * ks * 2, 256)
    return _align(off + 1152 * 4, 256)


def _ws_bytes(n, g0, d, B, H, W, train=False, x3=0):
    h, w, P = H // 2, W // 2, g0 // 8
    planes = [_align(12 * n, 32) // 8, P, P, P * d, 16 * d if train else 16, P, P]
    off = 0
    for p in planes:
        off = _align(off + B * p * (2 if x3 else 1) * h * w * 16, 256)
    return _align(off + B * 8 * (2 if x3 else 1) * H * W * 16, 256)


def _header_arch(tmp_path, cases):
    """BIN_BACKBONE_ARCH as a C compiler expands it from include/bin_b200.h."""
    lines = ['#include <stdio.h>', '#include "bin_b200.h"', 'int main(void) {']
    lines += [f'  printf("%d\\n", BIN_BACKBONE_ARCH({n}, {g0}, {d}));' for n, g0, d in cases] + ['  return 0;', '}']
    src, exe = tmp_path / "arch.c", tmp_path / "arch"
    src.write_text("\n".join(lines))
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    return [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]


def test_arch_encoding(tmp_path):
    from bin_b200 import _lib
    cases = [(n, g0, d) for n in (2, 3, 5) for g0, d in [(0, 0), (64, 6), (64, 1), (96, 12), (64, 12), (96, 6)]]
    assert _header_arch(tmp_path, cases) == [_lib.backbone_arch(*c) for c in cases]
    assert [_lib.backbone_arch(n, 0, 0) for n in (2, 3, 5)] == [2, 3, 5]


@pytest.mark.parametrize("g0,d", [(96, 12), (64, 6), (64, 1), (64, 12), (96, 6), (96, 1)])
@pytest.mark.parametrize("n", [2, 3, 5])
def test_size_queries_match_hand_computed_layouts(n, g0, d):
    from bin_b200 import _lib
    L = _lib.lib()
    a = _arch(n, g0, d)
    assert L.bin_backbone_nconv(a) == 5 * d + 6
    assert L.bin_backbone_packed_bytes(a) == L.bin_backbone_packed_bytes_p(a, 0) == _packed_bytes(n, g0, d)
    assert L.bin_backbone_packed_bytes_p(a, 1) == _packed_bytes(n, g0, d, x3=1)
    assert L.bin_backbone_packed_t_bytes(a) == _packed_t_bytes(n, g0, d)
    assert L.bin_backbone_grad_param_floats(a) == sum(co * ci * k * k + co for ci, co, k, _ in _convs(n, g0, d))
    for B, H, W in [(1, 64, 96), (6, 20, 36)]:
        assert L.bin_backbone_workspace_bytes(a, B, H, W) == _ws_bytes(n, g0, d, B, H, W)
        assert L.bin_backbone_workspace_bytes_p(a, B, H, W, 1) == _ws_bytes(n, g0, d, B, H, W, x3=1)
        assert L.bin_backbone_train_workspace_bytes(a, B, H, W) == _ws_bytes(n, g0, d, B, H, W, train=True)
        assert L.bin_backbone_grad_workspace_bytes(a, B, H, W) > 0
    if (g0, d) == (96, 12):                                   # the shipped arch is the frame count itself
        assert L.bin_backbone_packed_bytes(n) == L.bin_backbone_packed_bytes(a) and L.bin_backbone_nconv(n) == 66


def test_no_arch_needs_more_than_the_shipped_one():
    """D <= 12 and G0 <= 96: no table, mask or workspace grows beyond what the shipped configuration needs."""
    from bin_b200 import _lib
    L = _lib.lib()
    for n in (2, 3, 5):
        for g0 in (64, 96):
            for d in range(1, 13):
                a = _arch(n, g0, d)
                assert L.bin_backbone_nconv(a) <= _lib.BIN_BACKBONE_NCONV
                assert L.bin_backbone_workspace_bytes(a, 2, 64, 64) <= L.bin_backbone_workspace_bytes(n, 2, 64, 64)
                assert L.bin_backbone_train_workspace_bytes(a, 2, 64, 64) <= L.bin_backbone_train_workspace_bytes(n, 2, 64, 64)
                assert L.bin_backbone_grad_workspace_bytes(a, 2, 64, 64) <= L.bin_backbone_grad_workspace_bytes(n, 2, 64, 64)


# ------------------------------------------------------------------ everything else is refused
BAD_ARCHS = [(4, 0, 0), (2, 32, 6), (2, 128, 6), (3, 64, 13), (5, 96, 13), (2, 65, 6), (2, 64, 255)]


@pytest.mark.parametrize("kw", [dict(G0=32), dict(G0=128), dict(D=0), dict(D=13), dict(C=3), dict(G=16), dict(G0=64, D=6.0)])
def test_python_rejects_unsupported_configurations(kw):
    from bin_b200 import rdn
    from bin_b200._lib import BinB200Error
    for cls in CLASSES.values():
        with pytest.raises(BinB200Error, match="G0 in"):
            getattr(rdn, cls)(**kw)
    if "G0" in kw and "D" not in kw:
        with pytest.raises(BinB200Error):
            rdn.RDN_residual_interp_5_input(lstm=True, GO=kw["G0"])
        with pytest.raises(BinB200Error):
            rdn.RDB(growRate0=kw["G0"], growRate=32, nConvLayers=4)


def test_library_rejects_unsupported_archs_before_any_launch():
    """Every size query returns 0 (nconv: -1) and every entry point BIN_ERR_ARG for an arch outside G0 in {64, 96},
    D in 1..12.  The pointers are host addresses that are never dereferenced: a call that got as far as a launch would
    fail with BIN_ERR_CUDA (or crash) instead."""
    from bin_b200 import _lib
    L = _lib.lib()
    dummy = (C.c_float * 1024)()
    p = (C.addressof(dummy) + 255) // 256 * 256
    ptrs = (C.c_void_p * 66)(*([p] * 66))
    fr = _lib.Frames()
    fr.ncalls, fr.Bc = 1, 1
    for n, g0, d in BAD_ARCHS + [(2, 64, 6)]:
        fr.nframes = n
        a = _lib.backbone_arch(n, g0, d) if n != 4 else 4
        ok = (n, g0, d) == (2, 64, 6)
        assert (L.bin_backbone_nconv(a) == 36) if ok else (L.bin_backbone_nconv(a) == -1)
        if ok:
            continue
        for q in (L.bin_backbone_packed_bytes(a), L.bin_backbone_packed_t_bytes(a), L.bin_backbone_packed_bytes_p(a, 1),
                  L.bin_backbone_grad_param_floats(a), L.bin_backbone_workspace_bytes(a, 1, 64, 64),
                  L.bin_backbone_workspace_bytes_p(a, 1, 64, 64, 0), L.bin_backbone_train_workspace_bytes(a, 1, 64, 64),
                  L.bin_backbone_grad_workspace_bytes(a, 1, 64, 64)):
            assert q == 0, (a, q)
        big = 1 << 40
        calls = {
            "pack": lambda: L.bin_backbone_pack(a, ptrs, ptrs, p, None),
            "pack_p": lambda: L.bin_backbone_pack_p(a, ptrs, ptrs, p, 1, None),
            "pack_t": lambda: L.bin_backbone_pack_t(a, ptrs, p, None),
            "fwd": lambda: L.bin_backbone_fwd(a, p, C.byref(fr), 64, 64, p, big, None),
            "fwd_p": lambda: L.bin_backbone_fwd_p(a, p, C.byref(fr), 64, 64, p, big, 0, None),
            "fwd_train": lambda: L.bin_backbone_fwd_train(a, p, C.byref(fr), 64, 64, p, big, None),
            "bwd_masked": lambda: L.bin_backbone_bwd_masked(a, p, C.byref(fr), C.byref(fr), 64, 64, p, p, big, p, p, 0,
                                                            None, None),
            "bwd_recompute_masked": lambda: L.bin_backbone_bwd_recompute_masked(a, p, p, C.byref(fr), C.byref(fr), 64, 64,
                                                                                p, big, p, big, p, p, 0, None, None),
            "rdb_fwd": lambda: L.bin_rdb_fwd(p, a, 0, p, p, 1, 8, 8, p, big, None),
        }
        for name, call in calls.items():
            rc = call()
            assert rc == 1, (name, (n, g0, d), rc, L.bin_last_error().decode())


def test_rdb_fwd_rejects_a_block_index_past_the_depth():
    from bin_b200 import _lib
    L = _lib.lib()
    dummy = (C.c_float * 64)()
    p = C.addressof(dummy)
    rc = L.bin_rdb_fwd(p, _lib.backbone_arch(2, 64, 6), 6, p, p, 1, 8, 8, p, 1 << 40, None)
    assert rc == 1 and L.bin_last_error().decode() == "rdb_fwd: bad nframes/index"


def test_grad_plan_takes_the_backbones_conv_count():
    from bin_b200 import rdn
    from bin_b200._lib import BinB200Error
    from bin_b200.autograd import grad_plan
    m = rdn.RDN_residual_interp_2_1_input(G0=64, D=3)
    nconv, n, ncalls = m.nconv, 3, 2
    params = [i % 3 == 0 for i in range(2 * nconv)]
    need, frames = grad_plan((False, False) + (True,) * (ncalls * n) + tuple(params), ncalls, n, nconv)
    assert len(need) == 2 * nconv == 42 and list(need) == [int(x) for x in params]
    assert frames == [[True] * n] * ncalls
    with pytest.raises(BinB200Error, match="grad_plan"):
        grad_plan((False, False) + (True,) * (ncalls * n + 2 * nconv), ncalls, n)
