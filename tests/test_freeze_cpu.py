"""Frozen tensors (requires_grad False) without a device: the mapping from autograd's needs_input_grad to the masked
backward's 132-byte mask and frame table, the masked entry points' argument checks, the calls that ask for nothing
(they must return before touching a device), and which path each entry point takes when part of the net is frozen."""
import ctypes as C

import pytest
import torch

from oracle import bin_oracle as O

NCONV = 66


@pytest.fixture(scope="module")
def L():
    from bin_b200 import _lib
    assert _lib.ABI_VERSION == 6
    return _lib.lib()


def _err(L, rc):
    return rc, L.bin_last_error().decode()


def test_grad_plan_maps_needs_input_grad():
    from bin_b200.autograd import grad_plan
    ncalls, n = 2, 3
    frames = [True, False, False, False, False, True]
    params = [False] * (2 * NCONV)
    params[0] = True                          # SFENet1.weight
    params[2 * 65 + 1] = True                 # UPNet.2.bias
    params[2 * 7] = True                      # RDBs.1.convs.0 weight
    need, frame_needed = grad_plan((False, False, *frames, *params), ncalls, n)
    assert len(need) == 2 * NCONV and C.sizeof(need) == 132
    assert [i for i, v in enumerate(need) if v] == [0, 14, 131]
    assert frame_needed == [[True, False, False], [False, False, True]]
    need, frame_needed = grad_plan((False, False) + (False,) * (6 + 2 * NCONV), ncalls, n)
    assert not any(need) and frame_needed == [[False] * 3] * 2


def test_grad_plan_rejects_a_wrong_input_count():
    from bin_b200 import BinB200Error
    from bin_b200.autograd import grad_plan
    with pytest.raises(BinB200Error, match="grad_plan"):
        grad_plan((False, False) + (True,) * (5 + 2 * NCONV), 2, 3)


def test_grad_frames_table_has_null_for_frames_without_gradient():
    from bin_b200.autograd import _grad_frames
    a, b = torch.zeros(2, 3, 4, 4), torch.zeros(2, 3, 4, 4)
    fr = _grad_frames([[a, None], [None, b]], 2)
    assert (fr.ncalls, fr.nframes, fr.Bc) == (2, 2, 2)
    assert fr.frame[0][0] == a.data_ptr() and fr.frame[1][1] == b.data_ptr()
    assert fr.frame[0][1] is None and fr.frame[1][0] is None


def _tables(ncalls, n, Bc, frames_ptr):
    from bin_b200 import _lib
    dout, dfr = _lib.Frames(), _lib.Frames()
    for f in (dout, dfr):
        f.ncalls, f.nframes, f.Bc = ncalls, n, Bc
    for k in range(ncalls):
        for i in range(n):
            dfr.frame[k][i] = frames_ptr
    return dout, dfr


def test_masked_backward_argument_checks(L):
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    n, ncalls, Bc, H, W = 3, 2, 1, 32, 48
    gws = L.bin_backbone_grad_workspace_bytes(n, ncalls * Bc, H, W)
    dout, dfr = _tables(ncalls, n, Bc, p)
    none = (C.c_ubyte * 132)()
    one = (C.c_ubyte * 132)(*([0] * 131 + [1]))
    # grad_params may be NULL only when no parameter gradient is asked for
    rc = L.bin_backbone_bwd_masked(n, p, C.byref(dout), C.byref(dfr), H, W, p, p, gws, None, p, 0, None, None)
    assert _err(L, rc) == (1, "backbone_bwd: null argument")
    rc = L.bin_backbone_bwd_masked(n, p, C.byref(dout), C.byref(dfr), H, W, p, p, gws, None, p, 0, one, None)
    assert _err(L, rc) == (1, "backbone_bwd: null argument")
    rc = L.bin_backbone_bwd_masked(n, p, C.byref(dout), C.byref(dfr), H, W, p, p, gws, p, p, 2, none, None)
    assert _err(L, rc) == (1, "backbone_bwd: unknown flags")
    rc = L.bin_backbone_bwd_masked(n, p, C.byref(dout), C.byref(dfr), H, W, p, p, gws - 1, p, p, 0, none, None)
    assert _err(L, rc) == (4, "backbone_bwd: gradient workspace too small")
    fwd = L.bin_backbone_workspace_bytes(n, ncalls * Bc, H, W)
    rc = L.bin_backbone_bwd_recompute_masked(n, p, p, C.byref(dout), C.byref(dfr), H, W, p + 4, fwd, p, gws, p, p, 0,
                                             none, None)
    assert _err(L, rc) == (1, "backbone_bwd: forward workspace must be 256-byte aligned")
    rc = L.bin_backbone_bwd_recompute_masked(n, None, p, C.byref(dout), C.byref(dfr), H, W, p, fwd, p, gws, p, p, 0,
                                             none, None)
    assert _err(L, rc) == (1, "backbone_bwd: null argument")


def test_masked_backward_that_asks_for_nothing_launches_nothing(L):
    """No parameter and no frame wants a gradient: the call returns BIN_OK before any CUDA call (on a machine without a
    device a launch would fail with BIN_ERR_CUDA)."""
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    n, ncalls, Bc, H, W = 5, 2, 1, 32, 48
    gws = L.bin_backbone_grad_workspace_bytes(n, ncalls * Bc, H, W)
    dout, dfr = _tables(ncalls, n, Bc, None)
    none = (C.c_ubyte * 132)()
    for flags in (0, 1):
        rc = L.bin_backbone_bwd_masked(n, p, C.byref(dout), C.byref(dfr), H, W, p, p, gws, None, p, flags, none, None)
        assert _err(L, rc)[0] == 0
        fwd = L.bin_backbone_workspace_bytes(n, ncalls * Bc, H, W)
        aligned = (p + 255) // 256 * 256
        rc = L.bin_backbone_bwd_recompute_masked(n, p, p, C.byref(dout), C.byref(dfr), H, W, aligned, fwd, p, gws, None,
                                                 p, flags, none, None)
        assert _err(L, rc)[0] == 0


def test_convlstm_backward_outputs_may_be_null(L):
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    B, H, W = 2, 16, 24
    # nothing asked for: no launch, and no scratch needed in deterministic mode
    for flags in (0, 1):
        rc = L.bin_convlstm_bwd_ex(p, None, None, p, p, p, None, p, None, None, None, None, None, B, H, W, flags, None, 0,
                                   None)
        assert _err(L, rc)[0] == 0
    # the weight pass still needs its scratch in deterministic mode when dw or db is wanted
    rc = L.bin_convlstm_bwd_ex(p, None, None, p, p, p, None, p, None, None, None, None, p, B, H, W, 1, None, 0, None)
    assert _err(L, rc) == (1, "convlstm_bwd: BIN_DETERMINISTIC needs a scratch buffer")
    rc = L.bin_convlstm_bwd_ex(p, None, None, None, p, p, None, p, p, None, None, p, p, B, H, W, 0, None, 0, None)
    assert _err(L, rc) == (1, "convlstm_bwd: null argument")


@pytest.fixture(scope="module")
def cpu_net():
    from bin_b200 import rdn
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(0), strict=True)
    return m


@pytest.fixture
def routes(monkeypatch):
    """Replace the autograd entry functions with recorders, so the path an entry point picks shows without a device."""
    from bin_b200 import autograd
    seen = []
    for name in ("backbone_apply", "pyramid_apply", "pyramid3_apply", "convlstm_apply", "window_apply"):
        monkeypatch.setattr(autograd, name, lambda *a, _n=name, **k: seen.append(_n) or "grad")
    return seen


def _only_frozen(net, names):
    for k, p in net.named_parameters():
        p.requires_grad_(k not in names)


def test_entry_points_take_the_grad_path_when_any_read_tensor_trains(cpu_net, routes):
    net = cpu_net
    fr = O.synth_frames(6, 1, 16, 16)
    _only_frozen(net, {"model.model1_1.SFENet1.weight"})
    try:
        assert net.model.model1_1(fr[0], fr[1]) == "grad"
        assert net.model(*fr[:5]) == "grad"
        assert net.forward_pyramid3(*fr[:4]) == "grad"
        assert net(*fr) == "grad"
        _only_frozen(net, {"clstm_4_prime.Gates.weight"})                    # the bias alone still trains
        assert net.clstm_4_prime(fr[0], None) == "grad"
    finally:
        _only_frozen(net, set())
    assert routes == ["backbone_apply", "pyramid_apply", "pyramid3_apply", "window_apply", "convlstm_apply"]


def test_entry_points_take_the_inference_path_when_nothing_trains(cpu_net, routes):
    """Everything a call reads is frozen: the inference path (which refuses a CPU tensor) runs, not autograd."""
    from bin_b200 import BinB200Error
    net = cpu_net
    fr = O.synth_frames(6, 1, 16, 16)
    _only_frozen(net, {k for k, _ in net.named_parameters()})
    try:
        with pytest.raises(BinB200Error, match="CPU"):
            net.model.model1_1(fr[0], fr[1])
        with pytest.raises(BinB200Error, match="CPU"):
            net.forward_pyramid3(*fr[:4])
        # forward_pyramid3 reads model1_1..model3_1 only: a trainable model4_1 does not send it down the grad path
        net.model.model4_1.UPNet[2].bias.requires_grad_(True)
        with pytest.raises(BinB200Error, match="CPU"):
            net.forward_pyramid3(*fr[:4])
        assert net.model(*fr[:5]) == "grad"
    finally:
        _only_frozen(net, set())
    assert routes == ["pyramid_apply"]
