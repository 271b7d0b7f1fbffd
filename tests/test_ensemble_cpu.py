"""CPU checks of the x4 flip self-ensemble (rdn.set_self_ensemble, bin_flipx4_expand / bin_flipx4_mean): the oracle's
ensemble against the reference's own flipx4_forward (tests/golden/ensemble.npz), the C ABI's argument checks (no device
needed), mode validation, the unchanged state_dict, the errors raised before any device work, and the documented
test.py shim through the reference's own define_G."""
import ctypes as C
import hashlib
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import bin_oracle as O

ORIENTATIONS = [None, (-1,), (-2,), (-2, -1)]          # flipx4_forward's order (utils/test_util.py:119-130)


def oracle_flipx4(frames, sd):
    """utils/test_util.py:110-132 restated on the fp32 oracle, over all 6 frames and all 14 outputs."""
    acc = None
    for dims in ORIENTATIONS:
        outs = O.window_forward([f if dims is None else torch.flip(f, dims) for f in frames], sd)
        outs = [o if dims is None else torch.flip(o, dims) for o in outs]
        acc = outs if acc is None else [a + o for a, o in zip(acc, outs)]
    return [a / 4 for a in acc]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "ensemble.npz"))


@pytest.mark.parametrize("tag", ["a", "b"])
def test_oracle_ensemble_matches_the_reference_helper(golden, tag):
    B, H, W, seed = (int(v) for v in golden[f"{tag}_meta"])
    frames = O.synth_frames(6, B, H, W, seed=seed, smooth=True)
    assert hashlib.sha256(torch.stack(frames).numpy().tobytes()).hexdigest() == str(golden[f"{tag}_frames_sha256"])
    with torch.no_grad():
        got = torch.stack(oracle_flipx4(frames, O.synth_state_dict(0)))
        plain = torch.stack(O.window_forward(frames, O.synth_state_dict(0)))
    ref = torch.from_numpy(golden[f"{tag}_out"])
    assert got.shape == ref.shape == (14, B, 3, H, W)
    assert (got - ref).abs().max().item() <= 2e-6
    assert (plain - ref).abs().max().item() > 1e-3          # the ensemble is not the plain window


def test_flipx4_abi_rejects_bad_arguments_without_a_device():
    """bin_flipx4_expand / bin_flipx4_mean check every argument before their first CUDA call: each call here fails with
    BIN_ERR_ARG and its message (the pointers are fake and never dereferenced)."""
    from bin_b200 import _lib
    L = _lib.lib()
    buf = (C.c_float * 256)()
    p = [C.addressof(buf) + 64 * k for k in range(4)]
    tab = lambda *ptrs: (C.c_void_p * max(len(ptrs), 1))(*ptrs)          # noqa: E731
    cases = [  # (src table, dst table, n, B, H, W), error text
        ((None, tab(p[1]), 1, 1, 8, 8), "null table"),
        ((tab(p[0]), None, 1, 1, 8, 8), "null table"),
        ((tab(p[0]), tab(p[1]), 0, 1, 8, 8), "n must be 1..14"),
        ((tab(p[0]), tab(p[1]), 15, 1, 8, 8), "n must be 1..14"),
        ((tab(p[0]), tab(p[1]), -1, 1, 8, 8), "n must be 1..14"),
        ((tab(p[0]), tab(p[1]), 1, 0, 8, 8), "B, H and W must be >= 1"),
        ((tab(p[0]), tab(p[1]), 1, 1, 0, 8), "B, H and W must be >= 1"),
        ((tab(p[0]), tab(p[1]), 1, 1, 8, -2), "B, H and W must be >= 1"),
        ((tab(p[0]), tab(p[1]), 1, 1 << 30, 1 << 30, 1 << 30), "tensor too large"),
        ((tab(None), tab(p[1]), 1, 1, 8, 8), "null table entry"),
        ((tab(p[0], p[1]), tab(p[2], None), 2, 1, 8, 8), "null table entry"),
        ((tab(p[0]), tab(p[0]), 1, 1, 8, 8), "a dst equals a src"),
        ((tab(p[0], p[1]), tab(p[2], p[0]), 2, 1, 8, 8), "a dst equals a src"),
        ((tab(p[0], p[1]), tab(p[2], p[2]), 2, 1, 8, 8), "dst entries must be distinct"),
    ]
    for fname in ("bin_flipx4_expand", "bin_flipx4_mean"):
        fn = getattr(L, fname)
        for args, text in cases:
            rc = fn(*args, None)
            err = L.bin_last_error().decode()
            assert rc == 1 and text in err and err.startswith(fname[4:] + ":"), (fname, args[2:], rc, err)


def test_set_self_ensemble_validates_and_reaches_wrapped_nets():
    from bin_b200 import BinB200Error, rdn
    net = rdn.bin_stage4_lstm()
    for bad in ("flipx8", "FLIPX4", 4, True):
        with pytest.raises(BinB200Error, match="self-ensemble mode"):
            rdn.set_self_ensemble(net, bad)
    assert getattr(net, "self_ensemble", None) is None
    with pytest.raises(BinB200Error, match="no RDN_residual_interp_5_input_ConvLSTM_L"):
        rdn.set_self_ensemble(torch.nn.Sequential(torch.nn.Conv2d(3, 3, 3)), "flipx4")
    assert rdn.set_self_ensemble(net, "flipx4") is net and net.self_ensemble == "flipx4"
    assert all(getattr(m, "self_ensemble", None) is None for m in net.modules() if m is not net)
    rdn.set_self_ensemble(net, None)
    assert net.self_ensemble is None
    holder = torch.nn.Module()                              # a model object holding the net (bin_model.netG)
    holder.netG = torch.nn.DataParallel(net)
    rdn.set_self_ensemble(holder, "flipx4")
    assert net.self_ensemble == "flipx4"
    net.self_ensemble = "bogus"                             # set by hand: the forward refuses it
    with torch.no_grad(), pytest.raises(BinB200Error, match="self-ensemble mode"):
        net(*O.synth_frames(6, 1, 16, 16))


def test_state_dict_is_unchanged_by_the_mode(tmp_path):
    from bin_b200 import rdn
    plain, ens = rdn.bin_stage4_lstm(), rdn.set_self_ensemble(rdn.bin_stage4_lstm(), "flipx4")
    assert list(ens.state_dict().keys()) == list(plain.state_dict().keys()) and len(ens.state_dict()) == 1332
    assert len(list(ens.parameters())) == 540 and not list(ens.buffers())
    sd = O.synth_state_dict(4)
    res = ens.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    torch.save(ens.state_dict(), tmp_path / "ens.pth")
    back = rdn.bin_stage4_lstm()
    back.load_state_dict(torch.load(tmp_path / "ens.pth"), strict=True)
    assert all(torch.equal(a, b) for a, b in zip(back.state_dict().values(), sd.values()))
    assert ens.self_ensemble == "flipx4"


def test_ensemble_calls_fail_loudly_without_a_device():
    """No CPU fallback; a grad-enabled call and forward_pyramid3 are refused before any device work."""
    from bin_b200 import BinB200Error, ops, rdn
    net = rdn.set_self_ensemble(rdn.bin_stage4_lstm(), "flipx4")
    fr = O.synth_frames(6, 1, 16, 16)
    with torch.no_grad(), pytest.raises(BinB200Error, match="CUDA"):
        net(*fr)
    with pytest.raises(BinB200Error, match="inference-only"):
        net(*fr)                                            # the parameters require grad
    with torch.no_grad(), pytest.raises(BinB200Error, match="forward_pyramid3"):
        net.forward_pyramid3(*fr[:4])
    for fn in (ops.flipx4_expand, ops.flipx4_mean):
        with pytest.raises(BinB200Error, match="CUDA"):
            fn(fr)


def test_test_py_shim_sets_the_mode_through_define_g(monkeypatch):
    """INTEGRATION.md's recipe: with the shim in sys.modules, the reference's own models.networks.define_G builds a net
    with the ensemble on.  Needs a reference checkout named by BIN_REFERENCE; skipped without one."""
    ref = os.environ.get("BIN_REFERENCE", "")
    if not os.path.isfile(os.path.join(ref, "models", "networks.py")):
        pytest.skip("set BIN_REFERENCE to a checkout of the reference (laomao0/BIN) to run this test")
    for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
        monkeypatch.delitem(sys.modules, k)
    monkeypatch.syspath_prepend(ref)
    import bin_b200.rdn as R
    shim = types.ModuleType("models.archs.RDN")
    shim.__dict__.update(vars(R))
    shim.bin_stage4_lstm = lambda: R.set_self_ensemble(R.bin_stage4_lstm(), "flipx4")
    monkeypatch.setitem(sys.modules, "models.archs.RDN", shim)
    try:
        import models.archs                                 # noqa: F401  (the recipe's last line)
        import models.networks as networks
        netG = networks.define_G({"network_G": {"which_model_G": "bin_stage4", "nframes": 6, "version": 2}})
    finally:
        for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
            sys.modules.pop(k, None)
    assert isinstance(netG, R.RDN_residual_interp_5_input_ConvLSTM_L) and netG.self_ensemble == "flipx4"
    assert len(netG.state_dict()) == 1332
