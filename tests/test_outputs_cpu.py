"""CPU checks of the output selection (rdn.set_outputs): the live set read off the window schedule against one derived
from the fp32 oracle with autograd, the calls each selection costs per stage, argument checking, the attribute reaching
wrapped nets, the unchanged state_dict, and the refusals raised before any device work."""
import pytest
import torch

from oracle import bin_oracle as O

SELECTIONS = [(k,) for k in range(14)] + [(8, 12, 13), (4, 11), tuple(range(14))]


@pytest.fixture(scope="module")
def oracle_nodes():
    """Every backbone call and ConvLSTM image of one oracle window, by the schedule's node name, with the 14 outputs.
    The oracle runs the reference's 20 calls in its own order: step 0 is calls 0..9, step 1 calls 10..19, and the
    step-1 repeats of stage 1 (calls 10..12) are not nodes of the 17-call schedule."""
    names = {0: (1, 0), 1: (1, 1), 2: (1, 2), 3: (1, 3), 4: (2, 0), 5: (2, 1), 6: (2, 2), 7: (3, 0), 8: (3, 1), 9: (4, 0),
             13: (1, 4), 14: (2, 3), 15: (2, 4), 16: (2, 5), 17: (3, 2), 18: (3, 3), 19: (4, 1)}
    nodes, ncalls, ncells = {}, [0], [0]
    real_backbone, real_convlstm = O.backbone, O.convlstm

    def backbone(frames, sd, return_feats=False):
        out = real_backbone(frames, sd)
        if ncalls[0] in names:
            nodes[names[ncalls[0]]] = out
        ncalls[0] += 1
        return out

    def convlstm(x, sd, prefix, state=None):
        h, st = real_convlstm(x, sd, prefix, state)
        nodes[("lstm", ncells[0])] = h
        ncells[0] += 1
        return h, st

    frames = [f.requires_grad_(True) for f in O.synth_frames(6, 1, 8, 8, seed=2)]
    O.backbone, O.convlstm = backbone, convlstm
    try:
        outs = O.window_forward(frames, O.synth_state_dict(0))
    finally:
        O.backbone, O.convlstm = real_backbone, real_convlstm
    assert ncalls[0] == 20 and ncells[0] == 6 and len(nodes) == 23
    return nodes, outs


@pytest.mark.parametrize("wanted", SELECTIONS, ids=lambda w: "-".join(map(str, w)))
def test_live_set_equals_the_oracles_gradient_support(oracle_nodes, wanted):
    """A node is live when some wanted output has a gradient with respect to it that is not identically zero."""
    from bin_b200 import rdn
    nodes, outs = oracle_nodes
    keys = list(nodes)
    loss = sum(outs[i].sum() for i in wanted)
    grads = torch.autograd.grad(loss, [nodes[k] for k in keys], retain_graph=True, allow_unused=True)
    support = {k for k, g in zip(keys, grads) if g is not None and bool((g != 0).any())}
    assert rdn._window_live(wanted) == support
    assert all(rdn._OUT_NODE[i] in support for i in wanted)


@pytest.mark.parametrize("wanted,calls,cells", [((13, 8, 12), (4, 5, 3, 1), 6), ((9,), (4, 3, 2, 1), 0),
                                                ((10,), (1, 0, 0, 0), 0), (tuple(range(14)), (5, 6, 4, 2), 6)])
def test_calls_per_stage(wanted, calls, cells):
    from bin_b200 import rdn
    live = rdn._window_live(wanted)
    assert tuple(sum(1 for n in live if n[0] == s) for s in (1, 2, 3, 4)) == calls
    assert sum(1 for n in live if n[0] == "lstm") == cells


def test_schedule_passes_shortened_call_lists_and_skips_dead_cells():
    from types import SimpleNamespace
    from bin_b200 import rdn
    live = rdn._window_live((13, 8, 12))
    seen, cells = [], []

    def stage(model, calls):
        assert all(x is not None for c in calls for x in c)
        seen.append((model, len(calls)))
        return [f"{model}.{i}" for i in range(len(calls))]

    pyr = SimpleNamespace(model2_1="m2", model3_1="m3", model4_1="m4")
    lstm = lambda group: cells.append([k for k, _ in group]) or [f"p{k}" for k, _ in group]
    o = rdn._window_schedule(stage, lstm, pyr, ["F"] * 6, [None, "a", "b", "c", "d"], live)
    assert seen == [("m2", 5), ("m3", 3), ("m4", 1)] and cells == [[0, 1, 2], [3, 4], [5]]
    assert [i for i in range(14) if o[i] is not None] == [1, 2, 3, 5, 6, 8, 10, 11, 12, 13]
    seen.clear()
    o = rdn._window_schedule(stage, None, pyr, ["F"] * 6, [None] * 4 + ["d"], rdn._window_live((10,)))
    assert seen == [] and [i for i in range(14) if o[i] is not None] == [10]


def test_set_outputs_validates_and_reaches_wrapped_nets():
    from bin_b200 import BinB200Error, rdn
    net = rdn.bin_stage4_lstm()
    for bad in ((), [], (14,), (-1,), (3, 3), (1.0,), ("13",), (True,), 13, "8"):
        with pytest.raises(BinB200Error, match="set_outputs"):
            rdn.set_outputs(net, bad)
    for bad in ("zero", None, 0, "NONE"):
        with pytest.raises(BinB200Error, match="unwanted"):
            rdn.set_outputs(net, (13,), unwanted=bad)
    assert getattr(net, "outputs", None) is None
    with pytest.raises(BinB200Error, match="no RDN_residual_interp_5_input_ConvLSTM_L"):
        rdn.set_outputs(torch.nn.Sequential(torch.nn.Conv2d(3, 3, 3)), (13,))
    assert rdn.set_outputs(net, [13, 8, 12]) is net and net.outputs == ((8, 12, 13), "none")
    assert rdn.set_outputs(net, iter((9, 7)), unwanted="zeros").outputs == ((7, 9), "zeros")
    assert all(getattr(m, "outputs", None) is None for m in net.modules() if m is not net)
    rdn.set_outputs(net, None)
    assert net.outputs is None
    holder = torch.nn.Module()                              # a model object holding the net (bin_model.netG)
    holder.netG = torch.nn.DataParallel(net)
    rdn.set_outputs(holder, (13, 8, 12), unwanted="zeros")
    assert net.outputs == ((8, 12, 13), "zeros")
    net.outputs = (13, 8, 12)                               # set by hand: the forward refuses it
    with torch.no_grad(), pytest.raises(BinB200Error, match="output selection"):
        net(*O.synth_frames(6, 1, 16, 16))


def test_state_dict_is_unchanged_by_the_selection():
    from bin_b200 import rdn
    plain, sel = rdn.bin_stage4_lstm(), rdn.set_outputs(rdn.bin_stage4_lstm(), (13, 8, 12), unwanted="zeros")
    assert list(sel.state_dict().keys()) == list(plain.state_dict().keys()) and len(sel.state_dict()) == 1332
    assert len(list(sel.parameters())) == 540 and not list(sel.buffers())
    res = sel.load_state_dict(O.synth_state_dict(4), strict=True)
    assert not res.missing_keys and not res.unexpected_keys and sel.outputs == ((8, 12, 13), "zeros")


def test_selection_calls_fail_loudly_without_a_device():
    """No CPU fallback, and a grad-enabled call is refused before any device work."""
    from bin_b200 import BinB200Error, rdn
    net = rdn.set_outputs(rdn.bin_stage4_lstm(), (13, 8, 12))
    fr = O.synth_frames(6, 1, 16, 16)
    with torch.no_grad(), pytest.raises(BinB200Error, match="CUDA"):
        net(*fr)
    with pytest.raises(BinB200Error, match="inference-only"):
        net(*fr)                                            # the parameters require grad


def test_test_py_shim_sets_the_selection_through_define_g(monkeypatch):
    """INTEGRATION.md's recipe: with the shim in sys.modules, the reference's own models.networks.define_G builds a net
    with the selection on.  Needs a reference checkout named by BIN_REFERENCE; skipped without one."""
    import os
    import sys
    import types
    ref = os.environ.get("BIN_REFERENCE", "")
    if not os.path.isfile(os.path.join(ref, "models", "networks.py")):
        pytest.skip("set BIN_REFERENCE to a checkout of the reference (laomao0/BIN) to run this test")
    for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
        monkeypatch.delitem(sys.modules, k)
    monkeypatch.syspath_prepend(ref)
    import bin_b200.rdn as R
    shim = types.ModuleType("models.archs.RDN")
    shim.__dict__.update(vars(R))
    shim.bin_stage4_lstm = lambda: R.set_outputs(R.bin_stage4_lstm(), (13, 8, 12), unwanted="zeros")
    monkeypatch.setitem(sys.modules, "models.archs.RDN", shim)
    try:
        import models.archs                                 # noqa: F401  (the recipe's last line)
        import models.networks as networks
        netG = networks.define_G({"network_G": {"which_model_G": "bin_stage4", "nframes": 6, "version": 2}})
    finally:
        for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
            sys.modules.pop(k, None)
    assert isinstance(netG, R.RDN_residual_interp_5_input_ConvLSTM_L) and netG.outputs == ((8, 12, 13), "zeros")
    assert len(netG.state_dict()) == 1332
