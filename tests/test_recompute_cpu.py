"""Activation recomputation without a device: the set_activation_checkpointing switch and the argument checks of
bin_backbone_bwd_recompute (every call here is invalid and must fail before anything reaches a device)."""
import ctypes as C

import pytest
import torch

from oracle import bin_oracle as O


@pytest.fixture(scope="module")
def net():
    from bin_b200 import rdn
    torch.manual_seed(0)
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(0), strict=True)
    return m


class _Holder(torch.nn.Module):
    """Holds the net as `.module`, as nn.DataParallel does (bin_model.py:42), without moving it to a device."""

    def __init__(self, m):
        super().__init__()
        self.module = m


def test_switch_propagates_and_keeps_the_state_dict(net):
    from bin_b200 import rdn
    before = {k: v.clone() for k, v in net.state_dict().items()}
    wrapped = _Holder(net)
    try:
        assert rdn.set_activation_checkpointing(wrapped, "recompute") is wrapped
        assert all(m.activation_checkpointing == "recompute" for m in net.modules())
        assert rdn._checkpointing_of(net.model.model3_1) == "recompute"
        after = net.state_dict()
        assert list(after.keys()) == list(before.keys()) and len(after) == 1332
        assert all(torch.equal(after[k], before[k]) for k in before)
    finally:
        rdn.set_activation_checkpointing(net, None)
    assert all(m.activation_checkpointing is None for m in net.modules())
    assert rdn._checkpointing_of(rdn.bin_stage4_lstm()) is None          # default: keep the activations


def test_unknown_mode_raises(net):
    from bin_b200 import BinB200Error, rdn
    for mode in ("Recompute", "checkpoint", True, 1):
        with pytest.raises(BinB200Error, match="activation checkpointing"):
            rdn.set_activation_checkpointing(net, mode)
    assert all(getattr(m, "activation_checkpointing", None) is None for m in net.modules())
    net.model.model1_1.activation_checkpointing = "sometimes"          # set by hand: refused when the mode is read
    try:
        with pytest.raises(BinB200Error, match="activation checkpointing"):
            rdn._checkpointing_of(net.model.model1_1)
    finally:
        net.model.model1_1.activation_checkpointing = None


def _frames(ncalls, nframes, Bc):
    from bin_b200 import _lib
    f = _lib.Frames()
    f.ncalls, f.nframes, f.Bc = ncalls, nframes, Bc
    return f


def test_bwd_recompute_rejects_bad_forward_workspace_before_any_launch():
    """A NULL, undersized or unaligned forward workspace fails with BIN_ERR_ARG / BIN_ERR_WORKSPACE.  The other pointers
    are host buffers that are never dereferenced: a call that got as far as a launch would fail with BIN_ERR_CUDA here."""
    from bin_b200 import _lib
    L = _lib.lib()
    n, ncalls, Bc, H, W = 3, 6, 2, 64, 96
    need = L.bin_backbone_workspace_bytes(n, ncalls * Bc, H, W)
    assert 0 < need < L.bin_backbone_train_workspace_bytes(n, ncalls * Bc, H, W)
    dummy = (C.c_float * 64)()
    p = C.addressof(dummy)
    aligned = (p + 255) // 256 * 256 + 4096                                 # a plausible, 256-byte aligned address
    dout, dfr = _frames(ncalls, n, Bc), _frames(ncalls, n, Bc)
    gws = L.bin_backbone_grad_workspace_bytes(n, ncalls * Bc, H, W)

    def call(fwd_ws, fwd_bytes, nframes=n, blob=p):
        rc = L.bin_backbone_bwd_recompute(nframes, blob, p, C.byref(dout), C.byref(dfr), H, W, fwd_ws, fwd_bytes, p, gws,
                                          p, p, None)
        return rc, L.bin_last_error().decode()

    assert call(None, need) == (1, "backbone_bwd: null argument")
    assert call(aligned, need, blob=None) == (1, "backbone_bwd: null argument")
    assert call(aligned, need - 1) == (4, "backbone_bwd: forward workspace too small")
    assert call(aligned, 0) == (4, "backbone_bwd: forward workspace too small")
    assert call(aligned + 16, need) == (1, "backbone_bwd: forward workspace must be 256-byte aligned")
    assert call(aligned, need, nframes=4) == (1, "backbone_bwd: nframes must be 2, 3 or 5")
    bad = _frames(ncalls, n, Bc + 1)
    rc = L.bin_backbone_bwd_recompute(n, p, p, C.byref(dout), C.byref(bad), H, W, aligned, need, p, gws, p, p, None)
    assert rc == 1 and L.bin_last_error().decode() == "backbone_bwd: bad call tables"
