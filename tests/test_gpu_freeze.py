"""Fine-tuning with part of the network frozen (requires_grad False, DESIGN.md §4g).

A frozen tensor gets no gradient and costs no work: the backbone backward skips the weight and bias gradients nobody
asked for and every data gradient that feeds only frozen convs, a stage none of whose inputs needs a gradient runs the
inference forward and keeps nothing, and the ConvLSTM backward skips the passes whose outputs are not wanted.  What still
runs is the launch the full backward makes, on the same operands, so under torch.use_deterministic_algorithms(True)
every gradient that is kept is torch.equal to the all-trainable step's."""
import pytest
import torch

from oracle import bin_oracle as O

pytestmark = pytest.mark.gpu
MODES = (None, "recompute")
B, H, W = 2, 64, 96

_P2_FROZEN = ("model.model2_1.SFENet1.", "model.model2_1.SFENet2.") + tuple(f"model.model2_1.RDBs.{i}." for i in range(6))
_M1_HEADS = ("model.model1_1.GFF.", "model.model1_1.UPNet.")
# stage 1, the ConvLSTM cells and model2_1 up to RDBs[6].convs.0 frozen: stage 2's frames need no gradient, so its walk
# stops inside RDB 6 (after conv 33's weight gradient), with no data gradient into that RDB's input
_LATE_FROZEN = ("model.model1_1.",) + _P2_FROZEN + ("model.model2_1.RDBs.6.convs.0.",)
_ONE_LFF_BIAS = "model.model2_1.RDBs.11.LFF.bias"
# name -> (is this parameter trainable?, indices of the six frames that require grad)
CONFIGS = {
    "stage1_frozen": (lambda k: not k.startswith("model.model1_1."), ()),
    "only_model4_1": (lambda k: k.startswith("model.model4_1."), ()),
    "only_convlstm": (lambda k: ".Gates." in k, ()),
    "partial_backbone": (lambda k: not k.startswith(_P2_FROZEN), ()),
    "biases_frozen": (lambda k: not k.endswith(".bias"), ()),
    "all_frozen_frames": (lambda k: False, (0, 1, 2, 3, 4, 5)),
    "convlstm_two_frames": (lambda k: ".Gates." in k, (1, 4)),
    # backward walks that stop partway (stage 1 after GFF.0; stage 2 inside RDB 6, or at RDB 11's LFF)
    "model1_1_heads_only": (lambda k: k.startswith(_M1_HEADS), ()),
    "model2_1_late_rdbs": (lambda k: not k.startswith(_LATE_FROZEN) and ".Gates." not in k, ()),
    "one_lff_bias": (lambda k: k == _ONE_LFF_BIAS, ()),
}


@pytest.fixture
def det():
    """torch's deterministic mode without the NaN fill of torch.empty; both restored afterwards."""
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(),
            torch.utils.deterministic.fill_uninitialized_memory)
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    yield
    torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
    torch.utils.deterministic.fill_uninitialized_memory = prev[2]


@pytest.fixture(scope="module")
def net():
    from bin_b200 import rdn
    m = rdn.bin_stage4_lstm()
    m.load_state_dict(O.synth_state_dict(0), strict=True)
    m = m.cuda().train()
    yield m
    rdn.set_activation_checkpointing(m, None)
    _freeze(m, lambda k: True)


@pytest.fixture(scope="module")
def data():
    fr = [f.cuda() for f in O.synth_frames(6, B, H, W, seed=101, smooth=True)]
    gt = [f.cuda() for f in O.synth_frames(14, B, H, W, seed=102, smooth=True)]
    return fr, gt


def _freeze(net, trainable):
    for k, p in net.named_parameters():
        p.requires_grad_(bool(trainable(k)))


def _step(net, fr, gt, frames_grad=(), call=None):
    """zero_grad, forward, fused L1 loss, backward; returns (loss, {name: grad or None}, [frame grad or None])."""
    from bin_b200.loss import pixel_loss
    net.zero_grad(set_to_none=True)
    f = [x.clone().requires_grad_(i in frames_grad) for i, x in enumerate(fr)]
    outs = net(*f) if call is None else call(f)
    outs = list(outs) if isinstance(outs, (tuple, list)) else [outs]
    loss, _ = pixel_loss(outs, gt[:len(outs)], "l1", cycle_pairs=None if call is None else ())
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: (None if p.grad is None else p.grad.clone()) for k, p in net.named_parameters()}
    return loss.detach().clone(), grads, [None if x.grad is None else x.grad.clone() for x in f]


_REF = {}


def _reference(net, data, mode):
    """The all-trainable step with every frame requiring grad, once per checkpointing mode."""
    from bin_b200 import rdn
    if mode not in _REF:
        rdn.set_activation_checkpointing(net, mode)
        _freeze(net, lambda k: True)
        _REF[mode] = _step(net, *data, frames_grad=range(6))
    return _REF[mode]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("config", list(CONFIGS))
def test_kept_gradients_are_bit_identical(det, net, data, config, mode):
    from bin_b200 import rdn
    loss_r, grads_r, fgrads_r = _reference(net, data, mode)
    trainable, frames = CONFIGS[config]
    rdn.set_activation_checkpointing(net, mode)
    _freeze(net, trainable)
    try:
        loss, grads, fgrads = _step(net, *data, frames_grad=frames)
    finally:
        _freeze(net, lambda k: True)
        rdn.set_activation_checkpointing(net, None)
    assert torch.equal(loss, loss_r), (loss.item(), loss_r.item())
    assert len(grads) == 540
    wrong_none = [k for k in grads if trainable(k) and grads[k] is None]
    assert not wrong_none, wrong_none[:8]
    leaked = [k for k in grads if not trainable(k) and grads[k] is not None]
    assert not leaked, leaked[:8]
    diff = [k for k in grads if trainable(k) and not torch.equal(grads[k], grads_r[k])]
    assert not diff, diff[:8]
    for i in range(6):
        if i in frames:
            assert torch.equal(fgrads[i], fgrads_r[i]), ("frame", i)
        else:
            assert fgrads[i] is None, ("frame", i)


# ---------------------------------------------------------------------------------------------------- launch counts
KERNELS = {"wgrad": "::wgrad_kernel", "bias": "::p8_bias_grad_kernel", "lstm_w": "::convlstm_bwd_weights_kernel",
           "tail": "::rdb_tail_kernel", "bwd": "::grad_out_to_p8_kernel", "conv": "::conv_igemm_kernel"}


def _launches(net, data, trainable, frames=()):
    """Kernel launches of one profiled step in the net's current checkpointing mode, by KERNELS key."""
    from torch.profiler import ProfilerActivity, profile
    _freeze(net, trainable)
    try:
        _step(net, *data, frames_grad=frames)                               # warm-up: packed caches, workspaces
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _step(net, *data, frames_grad=frames)
    finally:
        _freeze(net, lambda k: True)
    n = dict.fromkeys(KERNELS, 0)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            for key, frag in KERNELS.items():
                n[key] += frag in ev.name
    return n


@pytest.fixture(scope="module")
def counts(net, data):
    """Launch counts of the all-trainable step and of one step per single trainable backbone."""
    from bin_b200 import rdn
    rdn.set_activation_checkpointing(net, None)
    c = {"all": _launches(net, data, lambda k: True)}
    for m in ("model1_1", "model2_1", "model3_1", "model4_1"):
        c[m] = _launches(net, data, lambda k, m=m: k.startswith(f"model.{m}."))
    return c


def test_all_trainable_counts(counts):
    """The baseline: 4 stage backwards, all training forwards (no fused tail), 6 ConvLSTM weight passes; each stage's
    weight and bias launches add up to the whole step's."""
    a = counts["all"]
    assert a["bwd"] == 4 and a["tail"] == 0 and a["lstm_w"] == 6 and a["wgrad"] > 0 and a["bias"] > 0, a
    for key in ("wgrad", "bias"):
        assert sum(counts[m][key] for m in ("model1_1", "model2_1", "model3_1", "model4_1")) == a[key], (key, counts)
    assert counts["model3_1"]["wgrad"] == counts["model4_1"]["wgrad"]          # two 5-frame backbones


def test_only_model4_1_runs_one_stage_backward(counts):
    c = counts["model4_1"]
    assert c["bwd"] == 1 and c["lstm_w"] == 0, c
    assert c["tail"] == 36, c                                                 # stages 1-3: inference forward, 12 RDBs
    assert 0 < c["wgrad"] < counts["all"]["wgrad"] and c["bias"] == 66, c


def test_only_convlstm_skips_every_weight_gradient(net, data, counts):
    c = _launches(net, data, lambda k: ".Gates." in k)
    assert c["wgrad"] == 0 and c["bias"] == 0 and c["lstm_w"] == 6, c
    assert c["bwd"] == 3 and c["tail"] == 12, c                               # stage 1: no backward, inference forward
    a = counts["all"]
    assert c["conv"] < a["conv"], (c, a)


def test_partial_backbone_drops_the_frozen_convs(net, data, counts):
    frozen = lambda k: k.startswith(_P2_FROZEN)
    part = _launches(net, data, lambda k: not frozen(k))
    only = _launches(net, data, frozen)
    for key in ("wgrad", "bias"):
        assert part[key] == counts["all"][key] - only[key], (key, part, only, counts["all"])
    assert only["bias"] == 32 and only["bwd"] == 3, only                     # convs 0..31; stage 1 needs no backward


# conv_igemm launches per backbone call batch: a training forward runs 66 convs, an inference forward 42 (the last growth
# conv and the LFF of each RDB run as one fused tail), and a full backward 114 data gradients: 4 in the head (UPNet.2 ...
# GFF.0), 9 per RDB (the LFF's x and growth rows, x rows of the 4 growth convs, growth rows of convs 3..1), SFENet2 and
# SFENet1.  The all-trainable window's stage 1 has no frame to differentiate, so it skips SFENet1's: 113.
FWD_TRAIN, FWD_INF, DGRAD = 66, 42, 114


@pytest.mark.parametrize("config,mode,expect", [
    # stage 1 stops after GFF.0's weight gradient (3 data gradients); stages 2-4 need every data gradient
    ("model1_1_heads_only", None, dict(conv=FWD_TRAIN + 3 + 3 * (FWD_TRAIN + DGRAD), bias=4, tail=0)),
    # stage 1 runs inference; stage 2: the head, RDBs 11..7, then in RDB 6 only the growth-map dgrads of the LFF and of
    # convs 3 and 2 (no input gradient below conv 33)
    ("model2_1_late_rdbs", None, dict(conv=FWD_INF + FWD_TRAIN + (4 + 5 * 9 + 3) + 2 * (FWD_TRAIN + DGRAD), bias=33 + 132,
                                      tail=12)),
    # stage 2 stops at RDB 11's LFF bias: the head's 4 data gradients
    ("one_lff_bias", None, dict(conv=FWD_INF + FWD_TRAIN + 4 + 2 * (FWD_TRAIN + DGRAD), bias=1, wgrad=0, tail=12)),
    # recompute: every stage with a backward runs its inference forward twice; stage 2 rebuilds no growth maps (its LFF
    # bias reads only the output gradient), stages 3 and 4 rebuild 4 per RDB
    ("one_lff_bias", "recompute", dict(conv=FWD_INF + (2 * FWD_INF + 4) + 2 * (2 * FWD_INF + 12 * 4 + DGRAD), bias=1,
                                       wgrad=0, tail=12 * 7)),
])
def test_partial_walks_launch_only_the_needed_data_gradients(net, data, counts, config, mode, expect):
    from bin_b200 import rdn
    a = counts["all"]
    assert a["conv"] == 4 * FWD_TRAIN + 3 * DGRAD + (DGRAD - 1), a
    rdn.set_activation_checkpointing(net, mode)
    try:
        c = _launches(net, data, CONFIGS[config][0])
    finally:
        rdn.set_activation_checkpointing(net, None)
    assert {k: c[k] for k in expect} == expect, (config, mode, c, expect)
    assert c["conv"] < a["conv"]


def test_frozen_network_skips_parameter_work(net, data):
    c = _launches(net, data, lambda k: False, frames=(0, 1, 2, 3, 4, 5))
    assert c["wgrad"] == 0 and c["bias"] == 0 and c["lstm_w"] == 0 and c["bwd"] == 4, c


# ---------------------------------------------------------------------------------------------------- memory
def test_memory_of_stages_without_backward(net):
    """Only model4_1 trainable: stages 1-3 keep no training workspace, so the step's peak falls by at least their
    bin_backbone_train_workspace_bytes (5, 6 and 4 calls)."""
    from bin_b200 import _lib, rdn
    from bin_b200.loss import pixel_loss
    Bm, Hm, Wm = 2, 128, 128
    fr = [f.cuda() for f in O.synth_frames(6, Bm, Hm, Wm, seed=103, smooth=True)]
    gt = [f.cuda() for f in O.synth_frames(14, Bm, Hm, Wm, seed=104, smooth=True)]
    L = _lib.lib()
    S = sum(L.bin_backbone_train_workspace_bytes(n, Bm * calls, Hm, Wm) for n, calls in ((2, 5), (3, 6), (5, 4)))
    rdn.set_activation_checkpointing(net, None)
    configs = {"all": lambda k: True, "only4": lambda k: k.startswith("model.model4_1.")}

    def step():
        net.zero_grad(set_to_none=True)
        loss, _ = pixel_loss(net(*fr), gt, "l1")
        loss.backward()

    peaks = {}
    try:
        for name, tr in configs.items():                                     # warm-up of both: the shared workspace
            _freeze(net, tr)
            step()
        for name, tr in configs.items():
            _freeze(net, tr)
            net.zero_grad(set_to_none=True)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            step()
            torch.cuda.synchronize()
            peaks[name] = torch.cuda.max_memory_allocated()
    finally:
        _freeze(net, lambda k: True)
        net.zero_grad(set_to_none=True)
    assert peaks["all"] - peaks["only4"] >= S, (peaks, S)


# ---------------------------------------------------------------------------------------------------- entry points
@pytest.mark.parametrize("entry", ["backbone", "pyramid", "pyramid3"])
def test_entry_points_with_sfenet1_frozen(det, net, data, entry):
    """Only model1_1.SFENet1.weight frozen and no frame requiring grad: every entry point still trains the rest, with
    the all-trainable step's bits."""
    from bin_b200 import rdn
    fr, gt = data
    calls = {"backbone": (lambda f: net.model.model1_1(f[0], f[1]), ("model.model1_1.",)),
             "pyramid": (lambda f: net.model(*f[:5]), ("model.",)),
             "pyramid3": (lambda f: net.forward_pyramid3(*f[:4]), ("model.model1_1.", "model.model2_1.", "model.model3_1."))}
    call, reads = calls[entry]
    rdn.set_activation_checkpointing(net, None)
    frozen = "model.model1_1.SFENet1.weight"
    _, ref, _ = _step(net, fr, gt, call=call)
    _freeze(net, lambda k: k != frozen)
    try:
        _, grads, _ = _step(net, fr, gt, call=call)
    finally:
        _freeze(net, lambda k: True)
    read = [k for k in grads if k.startswith(reads)]
    assert grads[frozen] is None
    got = [k for k in read if k != frozen and grads[k] is not None]
    assert len(got) == len(read) - 1 and len(got) >= 131, (entry, len(got), len(read))
    diff = [k for k in got if not torch.equal(grads[k], ref[k])]
    assert not diff, diff[:8]


# ---------------------------------------------------------------------------------------------------- optimizer
def test_adam_leaves_frozen_parameters_alone(data):
    """Stage 1 frozen, both optimizers built over all 540 tensors: three steps of bin_b200.optim.Adam track
    torch.optim.Adam, the frozen tensors keep their bits, get no state and no version bump, and model1_1's packed
    weights stay cached."""
    from bin_b200 import rdn
    from bin_b200.loss import pixel_loss
    from bin_b200.optim import Adam
    fr, gt = data
    nets, opts, losses = {}, {}, {"a": [], "b": []}
    for tag in ("a", "b"):
        m = rdn.bin_stage4_lstm()
        m.load_state_dict(O.synth_state_dict(2), strict=True)
        m = m.cuda().train()
        _freeze(m, lambda k: not k.startswith("model.model1_1."))
        nets[tag] = m
        opts[tag] = (Adam if tag == "a" else torch.optim.Adam)(m.parameters(), lr=1e-4, betas=(0.9, 0.99))
    frozen = {t: [p for k, p in nets[t].named_parameters() if k.startswith("model.model1_1.")] for t in nets}
    before = [p.detach().clone() for p in frozen["a"]]
    versions = [p._version for p in frozen["a"]]
    blob = nets["a"].model.model1_1.packed_blob()
    for _ in range(3):
        for tag in ("a", "b"):
            opts[tag].zero_grad(set_to_none=True)
            loss, _ = pixel_loss(nets[tag](*fr), gt, "l1")
            loss.backward()
            opts[tag].step()
            losses[tag].append(loss.item())
    torch.cuda.synchronize()
    assert losses["a"][2] < losses["a"][0]
    for x, y in zip(losses["a"], losses["b"]):
        assert abs(x - y) <= 2e-3 * abs(y), losses
    for tag in ("a", "b"):
        assert all(p.grad is None and len(opts[tag].state[p]) == 0 for p in frozen[tag])
        assert all(torch.equal(p, q) for p, q in zip(frozen[tag], before))
    assert [p._version for p in frozen["a"]] == versions
    assert nets["a"].model.model1_1.packed_blob() is blob
    trained = [p for k, p in nets["a"].named_parameters() if not k.startswith("model.model1_1.")]
    assert all(len(opts["a"].state[p]) == 3 for p in trained)
